"""GroupNorm and the GroupNorm ResNet-18 without a GPU: config and CLI acceptance and refusals, the
model's parameter spec, net / config agreement, the checkpoint refusal across norms, the layer's
forward and backward formulas (as the kernels evaluate them) against fp64 autograd, and ptxas on the
group-norm kernels."""
import re
import shutil
import subprocess
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as TF

from bflc_demo_b200 import build
from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.models.lora import check_net_matches_config
from bflc_demo_b200.models.nets import ResNet18, build_model
from bflc_demo_b200.ops.nn import GN_EPS, GN_GROUPS

F64 = torch.float64


# ------------------------------------------------------------------ config and CLI
def test_config_accepts_group_norm_for_resnet18_only():
    c = FLConfig(model="resnet18", resnet_norm="group").validate()
    assert FLConfig.from_json(c.to_json()) == c
    assert FLConfig().resnet_norm == "batch"
    FLConfig(model="resnet18", resnet_norm="batch").validate()
    for model in ("mlp", "lenet5", "bert", "gpt"):
        with pytest.raises(ValueError, match="resnet_norm applies to resnet18 only"):
            FLConfig(model=model, resnet_norm="group").validate()
    with pytest.raises(ValueError, match="resnet_norm must be batch or group"):
        FLConfig(model="resnet18", resnet_norm="layer").validate()


@pytest.mark.parametrize("argv, why", [
    (["--model", "lenet5", "--resnet-norm", "group"], "--resnet-norm applies to --model resnet18 only"),
    (["--model", "mlp", "--resnet-norm", "batch"], "--resnet-norm applies to --model resnet18 only"),
    (["--model", "gpt", "--resnet-norm", "group"], "--resnet-norm applies to --model resnet18 only"),
    (["--model", "resnet18", "--resnet-norm", "layer"], "invalid choice"),
])
def test_cli_refuses(argv, why, capsys):
    from bflc_demo_b200.run import main
    with pytest.raises(SystemExit) as e:
        main(argv)
    assert e.value.code == 2
    assert why in capsys.readouterr().err


# ------------------------------------------------------------------ the model
def test_group_norm_spec_drops_running_statistics_and_keeps_the_batch_spec():
    bn, gn = ResNet18(10), ResNet18(10, norm="group")
    assert bn.norm == "batch" and gn.norm == "group"
    bn_names = [e.name for e in bn.spec.entries]
    gn_names = [e.name for e in gn.spec.entries]
    assert gn_names == [n for n in bn_names if not n.endswith((".rmean", ".rvar"))]
    assert not any(n.endswith((".rmean", ".rvar")) for n in gn_names)
    # every norm of the batch spec still holds gamma, beta, rmean, rvar in that order
    for i, n in enumerate(bn_names):
        if n.endswith(".gamma"):
            stem = n[:-len(".gamma")]
            assert bn_names[i:i + 4] == [f"{stem}.{k}" for k in ("gamma", "beta", "rmean", "rvar")]
    n_stats = sum(e.numel for e in bn.spec.entries if e.name.endswith((".rmean", ".rvar")))
    assert sum(e.numel for e in gn.spec.entries) == sum(e.numel for e in bn.spec.entries) - n_stats
    assert gn.spec.total < bn.spec.total
    assert build_model("resnet18", 10).norm == "batch"
    assert build_model("resnet18", 10, norm="group").spec.total == gn.spec.total


def test_group_norm_genesis_has_unit_gamma_and_zero_beta():
    net = ResNet18(10, norm="group")
    master = torch.full((net.spec.total,), float("nan"))
    net.init_(master, seed=3)
    P = net.spec.views(master)
    gammas = [k for k in P if k.endswith(".gamma")]
    assert len(gammas) == 1 + 2 * 8 + 3
    for k in gammas:
        assert torch.equal(P[k], torch.ones_like(P[k]))
        assert torch.equal(P[k[:-len("gamma")] + "beta"], torch.zeros_like(P[k]))
    # the batch-norm model's genesis is unchanged by the option
    a, b = ResNet18(10), ResNet18(10, norm="batch")
    ma, mb = torch.empty(a.spec.total), torch.empty(b.spec.total)
    a.init_(ma, seed=3)
    b.init_(mb, seed=3)
    assert torch.equal(ma, mb)


def test_model_refuses_bad_norms_and_widths():
    with pytest.raises(ValueError, match="norm must be one of batch, group"):
        ResNet18(10, norm="layer")
    with pytest.raises(ValueError, match="multiple of 32"):
        ResNet18(10, widths=(8, 16, 16, 32), norm="group")
    ResNet18(10, widths=(8, 16, 16, 32))          # batch norm takes any width
    ResNet18(10, widths=(32, 32, 64, 64), norm="group")


def test_engine_refuses_a_net_whose_norm_is_not_the_configs():
    gn, bn = ResNet18(10, norm="group"), ResNet18(10)
    check_net_matches_config(FLConfig(model="resnet18", resnet_norm="group"), gn)
    check_net_matches_config(FLConfig(model="resnet18"), bn)
    with pytest.raises(ValueError, match="disagree on ResNet-18's norm"):
        check_net_matches_config(FLConfig(model="resnet18"), gn)
    with pytest.raises(ValueError, match="disagree on ResNet-18's norm"):
        check_net_matches_config(FLConfig(model="resnet18", resnet_norm="group"), bn)


@pytest.mark.parametrize("saved, engine", [("batch", "group"), ("group", "batch")])
def test_checkpoint_of_one_norm_is_refused_by_the_other(tmp_path, saved, engine):
    from bflc_demo_b200.utils.checkpoint import load_checkpoint
    src, dst = ResNet18(10, norm=saved), ResNet18(10, norm=engine)
    path = tmp_path / "ck.pt"
    torch.save(dict(version=2, world=1, rank=0, n_params=src.spec.total,
                    config=FLConfig(model="resnet18", resnet_norm=saved).to_json()), path)
    with pytest.raises(ValueError, match="n_params"):
        load_checkpoint(str(path), SimpleNamespace(n_params=dst.spec.total, world=1))


# ------------------------------------------------------------------ the layer's formulas in fp64
def gn_kernel_math(x, gamma, beta, dy, residual, relu, groups=GN_GROUPS, per_row=False):
    """The forward and backward as k_gn_fwd / k_gn_bwd evaluate them, in fp64, on channels-last
    x [N, H, W, C]: -> y, dx, dres, dgamma, dbeta and the per-example partials pg, pb [N, C].
    ``per_row``: the modelled mistake of statistics per row (pixel) instead of per (example, group)."""
    N, H, W, Cc = x.shape
    cg = Cc // groups
    xg = x.reshape(N, H * W, groups, cg)
    if per_row:
        m = xg.mean(dim=3, keepdim=True)
        v = ((xg - m) ** 2).mean(dim=3, keepdim=True)
    else:
        m = xg.mean(dim=(1, 3), keepdim=True)
        v = ((xg - m) ** 2).mean(dim=(1, 3), keepdim=True)
    rs = 1.0 / torch.sqrt(v + GN_EPS)
    xh = ((xg - m) * rs).reshape(N, H * W, Cc)
    pre = xh * gamma + beta
    if residual is not None:
        pre = pre + residual.reshape(N, H * W, Cc)
    y = pre.clamp_min(0) if relu else pre
    g = dy.reshape(N, H * W, Cc) * ((y > 0) if relu else 1.0)
    pg, pb = (g * xh).sum(1), g.sum(1)
    gh = (g * gamma).reshape(N, H * W, groups, cg)
    xhg = xh.reshape(N, H * W, groups, cg)
    red = (1, 3) if not per_row else (3,)
    dx = rs * (gh - gh.mean(dim=red, keepdim=True) - xhg * (gh * xhg).mean(dim=red, keepdim=True))
    shp = (N, H, W, Cc)
    return (y.reshape(shp), dx.reshape(shp), g.reshape(shp), pg.sum(0), pb.sum(0), pg, pb)


def _torch_ref(x, gamma, beta, dy, residual, relu):
    xt = x.permute(0, 3, 1, 2).clone().requires_grad_(True)
    gt, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    rt = residual.permute(0, 3, 1, 2).clone().requires_grad_(True) if residual is not None else None
    o = TF.group_norm(xt, GN_GROUPS, gt, bt, eps=GN_EPS)
    if rt is not None:
        o = o + rt
    if relu:
        o = torch.relu(o)
    o.backward(dy.permute(0, 3, 1, 2))
    nhwc = lambda t: t.permute(0, 2, 3, 1)   # noqa: E731
    return (nhwc(o.detach()), nhwc(xt.grad), nhwc(rt.grad) if rt is not None else None, gt.grad, bt.grad)


def _fixture(N, H, W, Cc, seed):
    gen = torch.Generator().manual_seed(seed)
    # per-channel offsets and scales, so a group's statistics differ from any one row's
    x = torch.randn(N, H, W, Cc, generator=gen, dtype=F64) * (0.5 + torch.rand(Cc, generator=gen, dtype=F64)) \
        + 2.0 * torch.randn(Cc, generator=gen, dtype=F64)
    gamma = 1.0 + 0.3 * torch.randn(Cc, generator=gen, dtype=F64)
    beta = 0.2 * torch.randn(Cc, generator=gen, dtype=F64)
    dy = torch.randn(N, H, W, Cc, generator=gen, dtype=F64)
    res = torch.randn(N, H, W, Cc, generator=gen, dtype=F64)
    return x, gamma, beta, dy, res


@pytest.mark.parametrize("Cc, HW, relu, has_res", [(64, 4, True, True), (128, 8, False, True),
                                                    (96, 2, True, False), (512, 4, False, False)])
def test_kernel_formulas_match_fp64_autograd(Cc, HW, relu, has_res):
    x, gamma, beta, dy, res = _fixture(3, HW, HW, Cc, seed=Cc + HW)
    res = res if has_res else None
    y, dx, dres, dg, db, pg, pb = gn_kernel_math(x, gamma, beta, dy, res, relu)
    ry, rdx, rres, rdg, rdb = _torch_ref(x, gamma, beta, dy, res, relu)
    for a, b in ((y, ry), (dx, rdx), (dg, rdg), (db, rdb)) + (((dres, rres),) if has_res else ()):
        assert torch.allclose(a, b, rtol=1e-10, atol=1e-10), float((a - b).abs().max())
    # each example's own dgamma / dbeta: the layer's gradient is their sum, and each is what the
    # example alone would produce
    for n in range(3):
        sl = slice(n, n + 1)
        _, _, _, dgn, dbn = _torch_ref(x[sl], gamma, beta, dy[sl], res[sl] if has_res else None, relu)
        assert torch.allclose(pg[n], dgn, rtol=1e-10, atol=1e-10)
        assert torch.allclose(pb[n], dbn, rtol=1e-10, atol=1e-10)


def test_statistics_per_row_instead_of_per_example_and_group_fail_the_fixture():
    x, gamma, beta, dy, res = _fixture(2, 4, 4, 64, seed=5)
    ry, rdx, _, rdg, _ = _torch_ref(x, gamma, beta, dy, res, True)
    y, dx, _, dg, _, _, _ = gn_kernel_math(x, gamma, beta, dy, res, True, per_row=True)
    assert float((y - ry).abs().max()) > 0.1
    assert float((dg - rdg).abs().max()) > 0.1
    # and statistics over the whole batch (batch norm's) mix the examples
    y0 = gn_kernel_math(x[:1], gamma, beta, dy[:1], res[:1], True)[0]
    assert torch.allclose(y0, gn_kernel_math(x, gamma, beta, dy, res, True)[0][:1], rtol=1e-12, atol=1e-12)
    bn = TF.batch_norm(x.permute(0, 3, 1, 2), None, None, gamma, beta, training=True, eps=GN_EPS)
    bn0 = TF.batch_norm(x[:1].permute(0, 3, 1, 2), None, None, gamma, beta, training=True, eps=GN_EPS)
    assert float((bn[:1] - bn0).abs().max()) > 0.1


# ------------------------------------------------------------------ ptxas
def test_group_norm_kernels_ptxas_clean(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(nvcc).exists():
        pytest.skip("nvcc not found")
    src = Path(build.CSRC) / "kernels" / "nn_kernels.cu"
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, "-I", str(Path(build.CSRC) / "include"), "-c", str(src),
           "-o", str(tmp_path / "n.o")]
    out = subprocess.run(cmd, capture_output=True, text=True, check=True)
    log = out.stdout + out.stderr
    blocks = re.findall(r"Function properties for (\w+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", log)
    gn = {name: props for name, *props in blocks if "k_gn_" in name}
    for k in ("k_gn_fwd", "k_gn_bwd", "k_gn_param"):
        hits = [p for name, p in gn.items() if k in name]
        assert len(hits) == 1, (k, list(gn))
        assert hits[0] == ["0", "0", "0"], (k, hits[0])
