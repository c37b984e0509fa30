"""DP-SGD for the convolutional families on the host: the dpsgd_conv opt-in and its refusals (config and CLI),
an fp64 specification of the convolution and group-norm sites checked against per-example fp64 autograd of
``conv2d`` / ``group_norm``, the norm-path rule on every LeNet-5 and ResNet-18 site, modelled mistakes that the
fixtures catch, and the ptxas report of the new kernels."""
import argparse
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from bflc_demo_b200 import build
from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.ops import dpsgd as D
from bflc_demo_b200.ops import gemm as G

F64 = torch.float64


# ------------------------------------------------------------------ config and CLI
def test_config_accepts_the_opt_in():
    for kw in (dict(model="lenet5"), dict(model="resnet18", resnet_norm="group")):
        c = FLConfig(dpsgd_clip=1.0, dpsgd_noise=1.0, dpsgd_conv=True, **kw).validate()
        assert c.dpsgd_on and c.dpsgd_conv
    assert not FLConfig().validate().dpsgd_conv


@pytest.mark.parametrize("kw, why", [
    (dict(model="lenet5", dpsgd_conv=True), "dpsgd_conv needs dpsgd_clip > 0"),
    (dict(model="mlp", dpsgd_clip=1.0, dpsgd_conv=True), "dpsgd_conv applies to lenet5 and resnet18, not mlp"),
    (dict(model="bert", lora_rank=8, dpsgd_clip=1.0, dpsgd_conv=True), "applies to lenet5 and resnet18, not bert"),
    (dict(model="resnet18", dpsgd_clip=1.0, dpsgd_conv=True), "batch norm mixes the examples"),
    (dict(model="lenet5", dtype="fp8", dpsgd_clip=1.0, dpsgd_conv=True), "dtype fp8 is not supported"),
    # without the opt-in the old refusals stand, naming the new alternative
    (dict(model="lenet5", dpsgd_clip=1.0), "does not cover lenet5"),
    (dict(model="resnet18", resnet_norm="group", dpsgd_clip=1.0), "does not cover resnet18"),
    (dict(model="lenet5", dpsgd_clip=1.0), "or opt in with dpsgd_conv"),
])
def test_config_refuses(kw, why):
    with pytest.raises(ValueError, match=re.escape(why)):
        FLConfig(**kw).validate()


@pytest.mark.parametrize("argv, why", [
    (["--model", "lenet5", "--dpsgd-conv"], "--dpsgd-conv needs --dpsgd-clip"),
    (["--model", "resnet18", "--dpsgd-clip", "1", "--dpsgd-conv"], "batch norm mixes the examples"),
    (["--model", "mlp", "--generic", "--dpsgd-clip", "1", "--dpsgd-conv"], "applies to lenet5 and resnet18"),
    (["--model", "lenet5", "--dtype", "fp8", "--dpsgd-clip", "1", "--dpsgd-conv"], "dtype fp8 is not supported"),
    (["--model", "lenet5", "--dpsgd-clip", "1"], "does not cover lenet5"),
    (["--model", "resnet18", "--resnet-norm", "group", "--dpsgd-clip", "1"], "does not cover resnet18"),
])
def test_cli_refuses(argv, why, capsys):
    from bflc_demo_b200.run import main
    with pytest.raises(SystemExit) as e:
        main(argv)
    assert e.value.code == 2
    assert why in capsys.readouterr().err


@pytest.mark.parametrize("model, norm", [("lenet5", None), ("resnet18", "group")])
def test_cli_accepts_the_opt_in(model, norm):
    from bflc_demo_b200.run import add_dpsgd_args, dpsgd_fields
    ap = argparse.ArgumentParser()
    add_dpsgd_args(ap)
    a = ap.parse_args(["--dpsgd-clip", "1", "--dpsgd-noise", "1", "--dpsgd-conv"])
    a.model, a.dtype, a.lora_rank, a.resnet_norm, a.generic, a.packed = model, "bf16", 0, norm, False, False
    kw = dpsgd_fields(ap, a)
    assert kw["dpsgd_conv"] and kw["dpsgd_clip"] == 1.0


def test_checkpoint_config_records_the_field():
    import json
    c = FLConfig(model="lenet5", dpsgd_clip=1.0, dpsgd_conv=True).validate()
    assert json.loads(c.to_json())["dpsgd_conv"] is True


# ------------------------------------------------------------------ fp64 specification
def patches(x: torch.Tensor, kh: int, kw: int, stride: int, pad: int) -> torch.Tensor:
    """x NHWC [N, H, W, C] -> the patch matrix [N, R, kh * kw * C], columns (tap r, tap t, channel) as the
    weights [Cout, kh * kw * Cin] are laid out; taps in the padding read 0."""
    N, H, W, Cc = x.shape
    xp = TF.pad(x.permute(0, 3, 1, 2), (pad, pad, pad, pad))
    u = TF.unfold(xp, (kh, kw), stride=stride)                     # [N, C * kh * kw, R], (c, r, t)
    R = u.shape[-1]
    return u.view(N, Cc, kh * kw, R).permute(0, 3, 2, 1).reshape(N, R, kh * kw * Cc)


def ones_col(P: torch.Tensor) -> torch.Tensor:
    return torch.cat([P, torch.ones(*P.shape[:-1], 1, dtype=P.dtype)], -1)


def sq_tiles(dz: torch.Tensor, P: torch.Tensor) -> torch.Tensor:
    """Per-example ||dz_n^T P_n||^2 as k_pe_norm forms it: 64 x 64 tiles of the product, each squared and
    reduced, the tiles summed."""
    V = dz.transpose(1, 2) @ P                                       # [N, a, b]
    a, b = V.shape[1:]
    return torch.stack([sum((V[n, i:i + 64, j:j + 64] ** 2).sum() for i in range(0, a, 64)
                            for j in range(0, b, 64)) for n in range(V.shape[0])])


def sq_gram(dz: torch.Tensor, P: torch.Tensor) -> torch.Tensor:
    """Per-example sum_{t,t'} (dz_t . dz_t') (p_t . p_t'), k_pe_gram's form."""
    return ((dz @ dz.transpose(1, 2)) * (P @ P.transpose(1, 2))).sum((1, 2))


def conv_per_example(x, w, b, dy, stride, pad):
    """fp64 autograd of torch's conv2d, one example at a time: (||dW_n||^2 + ||db_n||^2) [N]."""
    out = []
    for n in range(x.shape[0]):
        wn = w.clone().requires_grad_(True)
        bn = b.clone().requires_grad_(True) if b is not None else None
        y = TF.conv2d(x[n:n + 1], wn, bn, stride=stride, padding=pad)
        y.backward(dy[n:n + 1])
        out.append((wn.grad ** 2).sum() + ((bn.grad ** 2).sum() if bn is not None else 0.0))
    return torch.stack(out)


def conv_fixture(N, Cin, H, Cout, k, stride, pad, bias, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, Cin, H, H, generator=g, dtype=F64)
    w = torch.randn(Cout, Cin, k, k, generator=g, dtype=F64)
    b = torch.randn(Cout, generator=g, dtype=F64) if bias else None
    OH = (H + 2 * pad - k) // stride + 1
    dy = torch.randn(N, Cout, OH, OH, generator=g, dtype=F64)
    P = patches(x.permute(0, 2, 3, 1), k, k, stride, pad)
    dz = dy.permute(0, 2, 3, 1).reshape(N, OH * OH, Cout)
    return x, w, b, dy, P, dz


CASES = [  # N, Cin, H, Cout, k, stride, pad, bias
    (3, 3, 12, 6, 5, 1, 0, True),      # LeNet conv1 at a small image
    (2, 6, 7, 16, 5, 1, 0, True),      # LeNet conv2
    (2, 4, 8, 8, 3, 2, 1, False),      # stride 2 with padding
    (3, 8, 6, 5, 1, 2, 0, False),      # 1x1 stride-2 downsample
    (2, 70, 5, 3, 3, 1, 1, True),      # K past 64 and a bias column past a tile edge
]


@pytest.mark.parametrize("case", CASES)
def test_conv_site_norms_against_autograd(case):
    N, Cin, H, Cout, k, stride, pad, bias = case
    x, w, b, dy, P, dz = conv_fixture(*case)
    ref = conv_per_example(x, w, b, dy, stride, pad)
    Pb = ones_col(P) if bias else P
    torch.testing.assert_close(sq_tiles(dz, Pb), ref, rtol=1e-12, atol=1e-9)
    torch.testing.assert_close(sq_gram(dz, Pb), ref, rtol=1e-12, atol=1e-9)
    # the product of the two sides is the gradient itself, layout included
    for n in range(N):
        wn = w.clone().requires_grad_(True)
        TF.conv2d(x[n:n + 1], wn, None, stride=stride, padding=pad).backward(dy[n:n + 1])
        gw = wn.grad.permute(0, 2, 3, 1).reshape(Cout, -1)
        torch.testing.assert_close(dz[n].T @ P[n], gw, rtol=1e-12, atol=1e-9)


def patch_sq(x: torch.Tensor, kh: int, kw: int, stride: int, pad: int, clamp: bool = False) -> torch.Tensor:
    """||p_t||^2 per output position: the sum over the taps inside the image of ||x_pix||^2, padding 0 (clamp:
    the modelled mistake of reading the nearest edge pixel for a padding tap)."""
    N, H, W, _ = x.shape
    OH, OW = (H + 2 * pad - kh) // stride + 1, (W + 2 * pad - kw) // stride + 1
    px = (x ** 2).sum(-1)
    out = torch.zeros(N, OH, OW, dtype=x.dtype)
    for oh in range(OH):
        for ow in range(OW):
            for r in range(kh):
                for t in range(kw):
                    h, v = oh * stride + r - pad, ow * stride + t - pad
                    if clamp:
                        h, v = min(max(h, 0), H - 1), min(max(v, 0), W - 1)
                    elif not (0 <= h < H and 0 <= v < W):
                        continue
                    out[:, oh, ow] += px[:, h, v]
    return out.view(N, -1)


@pytest.mark.parametrize("case", CASES)
def test_patch_norm_formula_and_abs_term(case):
    N, Cin, H, Cout, k, stride, pad, bias = case
    x, w, b, dy, P, dz = conv_fixture(*case)
    xs = x.permute(0, 2, 3, 1)
    torch.testing.assert_close(patch_sq(xs, k, k, stride, pad), (P ** 2).sum(-1), rtol=1e-12, atol=0)
    # ab_n = sum_t ||dz_t|| ||(p_t, 1)|| bounds every example's gradient norm (Cauchy-Schwarz, row by row)
    ab = (dz.norm(dim=-1) * ((P ** 2).sum(-1) + float(bias)).sqrt()).sum(-1)
    assert (conv_per_example(x, w, b, dy, stride, pad).sqrt() <= ab * (1 + 1e-12)).all()


def gn_partials(x, dy, gamma, beta, G=4, eps=1e-5):
    """k_gn_bwd's per-example partials: pg[n, c] = sum_hw dy xhat, pb[n, c] = sum_hw dy (fp64)."""
    N, Cc, H, W = x.shape
    xg = x.view(N, G, -1)
    mean, var = xg.mean(-1, keepdim=True), xg.var(-1, unbiased=False, keepdim=True)
    xhat = ((xg - mean) / (var + eps).sqrt()).view_as(x)
    return (dy * xhat).sum((2, 3)), dy.sum((2, 3))


def gn_fixture(seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(3, 8, 4, 4, generator=g, dtype=F64)
    dy = torch.randn(3, 8, 4, 4, generator=g, dtype=F64)
    gamma, beta = torch.randn(8, generator=g, dtype=F64), torch.randn(8, generator=g, dtype=F64)
    ref = []
    for n in range(3):
        gm, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
        TF.group_norm(x[n:n + 1], 4, gm, bt, eps=1e-5).backward(dy[n:n + 1])
        ref.append((gm.grad ** 2).sum() + (bt.grad ** 2).sum())
    return x, dy, gamma, beta, torch.stack(ref)


def test_group_norm_partial_norms_against_autograd():
    x, dy, gamma, beta, ref = gn_fixture()
    pg, pb = gn_partials(x, dy, gamma, beta)
    torch.testing.assert_close((pg ** 2).sum(1) + (pb ** 2).sum(1), ref, rtol=1e-12, atol=1e-12)
    # the release with factors c: sum_n c_n pg_n, and each example's part has norm c_n sqrt(sq_n)
    c = torch.tensor([1.0, 0.5, 0.0], dtype=F64)
    rel = (c[:, None] * pg).sum(0)
    torch.testing.assert_close(rel, pg[0] + 0.5 * pg[1], rtol=1e-15, atol=0)


# path selection: a = Cout, b = the patch width with the bias column
LENET = [("conv1", 784, 8, 80 + 1), ("conv2", 100, 16, 200 + 1)]
RESNET = [("stem", 1024, 64, 32), ("l0.c", 1024, 64, 576), ("l1.0.c1", 256, 128, 576), ("l1.c2", 256, 128, 1152),
          ("l1.0.down", 256, 128, 64), ("l2.0.c1", 64, 256, 1152), ("l2.c2", 64, 256, 2304),
          ("l2.0.down", 64, 256, 128), ("l3.0.c1", 16, 512, 2304), ("l3.c2", 16, 512, 4608),
          ("l3.0.down", 16, 512, 256)]


def test_norm_path_rule_on_every_site():
    want = {"conv1": "tiles", "conv2": "tiles", "stem": "tiles", "l0.c": "tiles", "l1.0.c1": "tiles",
            "l1.c2": "tiles", "l1.0.down": "tiles", "l2.0.c1": "gram", "l2.c2": "gram", "l2.0.down": "gram",
            "l3.0.c1": "gram", "l3.c2": "gram", "l3.0.down": "gram"}
    for name, R, a, b in LENET + RESNET:
        assert D.conv_norm_path(R, a, b) == want[name], name
    # the rule is the operation count: Gram R^2 (a + b) per example against the tiles' R a b
    assert D.conv_norm_path(512, 10 ** 4, 10 ** 4) == "gram" and D.conv_norm_path(513, 10 ** 4, 10 ** 4) == "tiles"


def test_step_buffers_fit_the_conv_models():
    from bflc_demo_b200.models.nets import LeNet5, ResNet18
    for net in (LeNet5(), ResNet18(norm="group")):
        step = D.DPSGDStep(net.spec, 4, 1.0, 0.0, 0, torch.zeros(1, dtype=torch.int32), "cpu", conv=True)
        plain = D.DPSGDStep(net.spec, 4, 1.0, 0.0, 0, torch.zeros(1, dtype=torch.int32), "cpu")
        # the convolution tiles only where asked for (LeNet's fit the existing 136-row allowance already)
        assert plain.sq.shape[0] <= step.sq.shape[0] and (plain.sq.shape[0] < step.sq.shape[0]) == (net.norm == "group"
                                                                                                     if hasattr(net, "norm") else False)
        need = 0
        for e in net.spec.entries:
            if len(e.shape) == 2:
                a, k = e.shape
                need += ((a + 63) // 64) * ((k + 1 + 63) // 64)   # tiles with a bias column, the widest form
                if k % 64 == 0:                                     # the implicit-GEMM norm's 128 x 64 tiles
                    assert ((a + 127) // 128) * (k // 64) <= ((a + 63) // 64) * ((k + 1 + 63) // 64)
            else:
                need += 1
        assert step.sq.shape[0] >= need


def test_fixed_splits_hold_whole_examples_and_depend_on_shapes_only():
    for rows, n, k, groups in ((64 * 1024, 64, 576, 64), (64 * 16, 512, 4608, 64), (3 * 784, 8, 80, 3),
                               (128 * 784, 8, 80, 128), (1, 8, 8, 1)):
        s = G.fixed_splits(rows, n, k, groups)
        assert groups % s == 0 and s >= 1
        tiles = ((n + 127) // 128) * ((k + 127) // 128)
        assert s == 1 or (s * tiles <= G.FIXED_SPLIT_CTAS and rows // s >= 64 * 8)
    assert G.fixed_splits(64 * 1024, 64, 576, 64) == 16    # ResNet stage 1: 5 tiles, 16 whole-example slices
    # the implicit-GEMM release: every split a multiple of 64 pixels (R 16: at least 4 examples per split)
    s = G.fixed_splits(64 * 16, 512, 4608, 64, align=64)
    assert s >= 1 and 64 % s == 0 and (64 * 16 // s) % 64 == 0
    assert G.fixed_splits(3 * 16, 8, 64, 3, align=64) == 0


# ------------------------------------------------------------------ modelled mistakes
def test_fixture_catches_the_bias_column_omitted():
    x, w, b, dy, P, dz = conv_fixture(*CASES[0])
    ref = conv_per_example(x, w, b, dy, 1, 0)
    assert not torch.allclose(sq_tiles(dz, P), ref, rtol=1e-6)


def test_fixture_catches_padding_taps_counted():
    x, *_ = conv_fixture(*CASES[2])
    xs = x.permute(0, 2, 3, 1)
    assert not torch.allclose(patch_sq(xs, 3, 3, 2, 1, clamp=True), patch_sq(xs, 3, 3, 2, 1), rtol=1e-6)


def test_fixture_catches_a_pixel_block_spanning_examples():
    # R = 16 output positions per example: 64-pixel K blocks of the flat rows span four examples
    case = (4, 8, 4, 8, 3, 1, 1, False)
    x, w, b, dy, P, dz = conv_fixture(*case)
    ref = conv_per_example(x, w, b, dy, 1, 1)
    flat_dz, flat_p = dz.reshape(-1, dz.shape[-1]), P.reshape(-1, P.shape[-1])
    wrong = torch.zeros(4, dtype=F64)
    for k0 in range(0, flat_dz.shape[0], 64):          # each block charged to the example of its first row
        blk = flat_dz[k0:k0 + 64].T @ flat_p[k0:k0 + 64]
        wrong[k0 // 16] += (blk ** 2).sum()
    assert not torch.allclose(wrong, ref, rtol=1e-6)
    torch.testing.assert_close(sq_tiles(dz, P), ref, rtol=1e-12, atol=1e-9)


def clip_release(sites, clip: float, per_site: bool) -> torch.Tensor:
    """One example's released gradient over its sites [(flat fp64 gradient)], clipped as the specification
    does (one factor from the whole vector's norm) or, the modelled mistake, each site by its own norm."""
    if per_site:
        return torch.cat([g * min(1.0, clip / float(g.norm())) for g in sites])
    full = torch.cat(sites)
    return full * min(1.0, clip / float(full.norm()))


def test_fixture_catches_per_site_clipping():
    # one example with a convolution site (its fp64 weight and bias gradient) and a group-norm site (gamma, beta)
    x, w, b, dy, P, dz = conv_fixture(*CASES[0])
    wn, bn = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    TF.conv2d(x[:1], wn, bn, stride=1).backward(dy[:1])
    conv = torch.cat([wn.grad.flatten(), bn.grad])
    xg, dyg, gamma, beta, _ = gn_fixture()
    gm, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    TF.group_norm(xg[:1], 4, gm, bt, eps=1e-5).backward(dyg[:1])
    gn = torch.cat([gm.grad, bt.grad])
    clip = 0.5 * min(float(conv.norm()), float(gn.norm()))     # both sites above C on their own
    assert float(clip_release([conv, gn], clip, per_site=False).norm()) <= clip * (1 + 1e-12)
    wrong = float(clip_release([conv, gn], clip, per_site=True).norm())
    assert wrong > 1.4 * clip       # sqrt(2) C: per-site clipping releases more than C for this example


def test_fixture_catches_gn_partials_summed_before_squaring():
    x, dy, gamma, beta, ref = gn_fixture()
    pg, pb = gn_partials(x, dy, gamma, beta)
    wrong = ((pg.sum(0) ** 2).sum() + (pb.sum(0) ** 2).sum()).expand(3)
    assert not torch.allclose(wrong, ref, rtol=1e-6)


# ------------------------------------------------------------------ ptxas
def _ptxas(tmp_path, name):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(nvcc).exists():
        pytest.skip("nvcc not found")
    src = Path(build.CSRC) / "kernels" / name
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, "-I", str(Path(build.CSRC) / "include"), "-c", str(src),
           "-o", str(tmp_path / "k.o")]
    out = subprocess.run(cmd, capture_output=True, text=True, check=True)
    log = out.stdout + out.stderr
    return {name: props for name, *props in re.findall(
        r"Function properties for (\w+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
        log)}


def test_new_kernels_ptxas_clean(tmp_path):
    """The generalised k_pe_norm, the lifted k_pe_rows, the implicit sites' k_patch_rows, the group-norm norm and
    release kernels and the slice sum of the deterministic split-K: no stack frame, no spills.  The patch
    sites' split-K GEMM is the existing batched bf16 instantiation."""
    props = {**_ptxas(tmp_path, "dpsgd_kernels.cu"), **_ptxas(tmp_path, "nn_kernels.cu")}
    for k in ("k_pe_norm", "k_pe_rows", "k_patch_rows", "k_pe_gn", "k_sum_slices", "k_gn_param"):
        hits = [p for name, p in props.items() if k in name]
        assert len(hits) == 1, (k, sorted(props))
        assert hits[0] == ["0", "0", "0"], (k, hits[0])


def test_k_group_gemm_instantiation_ptxas_clean(tmp_path):
    """The implicit-GEMM weight gradient by K groups (gemm_kernel<64, 3>: per-example norms in the epilogue, or
    plain stores into workspace slices) is a new instantiation: no stack frame, no spills, and the existing
    instantiations stay clean."""
    props = _ptxas(tmp_path, "gemm_sm100.cu")
    hits = [p for name, p in props.items() if "gemm_kernelILi64ELi3E" in name]
    assert len(hits) == 1, sorted(props)
    for name, p in props.items():
        if "gemm_kernel" in name:
            assert p[1:] == ["0", "0"], (name, p)
    assert hits[0] == ["0", "0", "0"], hits[0]
