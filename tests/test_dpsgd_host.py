"""DP-SGD local training on the host: config and CLI refusals, the local accountant, the noise site word,
the host train_pass against brute-force per-example fp64 autograd, the fp32 clip-factor specification
with its certified bound, the new kernels' ptxas report, and modelled mistakes that the fixtures catch."""
import math
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from bflc_demo_b200 import build
from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.engine.generic import dpsgd_epsilon, resolve_dpsgd_seed
from bflc_demo_b200.host.models import HostDPSGD, HostModel
from bflc_demo_b200.ops import dpsgd as D
from bflc_demo_b200.protocol import oracle as O
from bflc_demo_b200.protocol import privacy

F32 = np.float32


# ------------------------------------------------------------------ config and CLI
def test_config_accepts_and_refuses():
    c = FLConfig(dpsgd_clip=1.0, dpsgd_noise=0.7, dpsgd_seed=3).validate()
    assert c.dpsgd_on and c.dpsgd_constants == (F32(1.0), F32(0.7))
    assert not FLConfig().validate().dpsgd_on
    assert FLConfig(model="gpt", lora_rank=8, dpsgd_clip=1.0).validate().dpsgd_on
    assert FLConfig(dpsgd_clip=1.0, dp_clip=2.0, dp_noise=1.0, prox_mu=0.1, server_opt="adam",
                    clip_grad_norm=1.0).validate().dpsgd_on
    bad = [dict(dpsgd_clip=-1.0), dict(dpsgd_clip=math.inf), dict(dpsgd_clip=1e39), dict(dpsgd_noise=1.0),
           dict(dpsgd_clip=1.0, dpsgd_noise=-1.0), dict(dpsgd_clip=1.0, dpsgd_noise=math.nan),
           dict(dpsgd_clip=1.0, dpsgd_seed=-1), dict(dpsgd_clip=1.0, dpsgd_seed=1 << 64),
           dict(dpsgd_clip=1.0, model="lenet5"), dict(dpsgd_clip=1.0, model="resnet18"),
           dict(dpsgd_clip=1.0, model="bert"), dict(dpsgd_clip=1.0, model="gpt"),
           dict(dpsgd_clip=1.0, dtype="fp8")]
    for kw in bad:
        with pytest.raises(ValueError):
            FLConfig(**kw).validate()


@pytest.mark.parametrize("argv, why", [
    (["--model", "mlp", "--dpsgd-clip", "1"], "fused MLP trainer has no per-example clipping"),
    (["--model", "lenet5", "--dpsgd-clip", "1"], "does not cover lenet5"),
    (["--model", "resnet18", "--dpsgd-clip", "1"], "does not cover resnet18"),
    (["--model", "bert", "--dpsgd-clip", "1"], "DP-SGD on bert needs LoRA"),
    (["--model", "gpt", "--dpsgd-clip", "1"], "DP-SGD on gpt needs LoRA"),
    (["--model", "bert", "--lora-rank", "8", "--packed", "--dpsgd-clip", "1"], "does not support --packed"),
    (["--model", "mlp", "--generic", "--dtype", "fp8", "--dpsgd-clip", "1"], "dtype fp8 is not supported"),
    (["--model", "mlp", "--generic", "--dpsgd-noise", "1"], "--dpsgd-noise / --dpsgd-seed need --dpsgd-clip"),
])
def test_cli_refuses(argv, why, capsys):
    from bflc_demo_b200.run import main
    with pytest.raises(SystemExit) as e:
        main(argv)
    assert e.value.code == 2
    assert why in capsys.readouterr().err


def test_engines_without_per_example_clipping_refuse():
    from bflc_demo_b200.engine.fused import FusedEngine
    from bflc_demo_b200.engine.nccl_baseline import NcclBaselineEngine
    cfg = FLConfig.for_world(1, dpsgd_clip=1.0)
    with pytest.raises(ValueError, match="DP-SGD"):
        FusedEngine(cfg, None)
    with pytest.raises(ValueError, match="DP-SGD"):
        NcclBaselineEngine(cfg, None)


def test_client_keys_are_secret_per_rank_or_derived_for_tests():
    cfg = FLConfig(dpsgd_clip=1.0, dpsgd_noise=1.0)
    assert resolve_dpsgd_seed(cfg, 0) != resolve_dpsgd_seed(cfg, 0)          # fresh secret bits
    t = FLConfig(dpsgd_clip=1.0, dpsgd_noise=1.0, dpsgd_seed=5)
    assert resolve_dpsgd_seed(t, 1) == resolve_dpsgd_seed(t, 1) != resolve_dpsgd_seed(t, 2)
    assert resolve_dpsgd_seed(FLConfig(dpsgd_clip=1.0), 0) == 0                # no noise: nothing draws


# ------------------------------------------------------------------ accounting and the site word
@pytest.mark.parametrize("opt_total, E, k", [(0, 4, 0), (1, 4, 1), (4, 4, 1), (5, 4, 2), (40, 4, 10), (7, 1, 7)])
def test_local_accountant(opt_total, E, k):
    cfg = FLConfig(dpsgd_clip=1.0, dpsgd_noise=1.3, dp_delta=1e-6)
    eps, delta = dpsgd_epsilon(cfg, opt_total, E)
    assert delta == 1e-6
    assert eps == (privacy.epsilon(float(F32(1.3)), k, 1e-6) if k else 0.0)
    assert dpsgd_epsilon(FLConfig(dpsgd_clip=1.0), opt_total, E)[0] == (math.inf if k else 0.0)


def test_site_words_are_separate():
    hdr = (Path(build.CSRC) / "include" / "consensus_math.hpp").read_text()
    assert int(re.search(r"kDpsgdSite = (0x[0-9A-F]+)u", hdr).group(1), 16) == O.DPSGD_SITE
    assert int(re.search(r"kDpSite = (0x[0-9A-F]+)u", hdr).group(1), 16) == O.DP_SITE
    assert O.DPSGD_SITE != O.DP_SITE and min(O.DPSGD_SITE, O.DP_SITE) >= 1 << 24
    a, b = O.dp_gauss(9, 3, 0, 64, O.DPSGD_SITE), O.dp_gauss(9, 3, 0, 64)
    assert not np.array_equal(a, b) and np.array_equal(b, O.dp_gauss(9, 3, 0, 64, O.DP_SITE))


# ------------------------------------------------------------------ the host path against fp64
def _brute(model, w, X, y, clip, noise, seed, step):
    """The definition in fp64: one autograd pass per example."""
    w64 = w.double()
    gs = []
    for n in range(X.shape[0]):
        wn = w64.clone().requires_grad_(True)
        p = model.spec.views(wn)
        x = X[n:n + 1].double() * model.scale
        h = torch.relu(x @ p["w1"].t() + p["b1"]) if model.kind == "mlp" else x
        logits = h @ (p["w2"] if model.kind == "mlp" else p["w"]).t() + (p["b2"] if model.kind == "mlp" else p["b"])
        gs.append(torch.autograd.grad(torch.nn.functional.cross_entropy(logits, y[n:n + 1].long()), wn)[0])
    g = torch.stack(gs)
    c = (clip / g.norm(dim=1)).clamp(max=1.0)
    xi = torch.from_numpy(O.dp_gauss(seed, step, 0, w.numel(), O.DPSGD_SITE)).double()
    return ((c[:, None] * g).sum(0) + noise * clip * xi) / X.shape[0]


@pytest.mark.parametrize("kind", ["softmax", "mlp"])
def test_host_train_pass_against_per_example_fp64(kind):
    torch.manual_seed(0)
    model = HostModel(kind, 12, 5, hidden=16)
    w = model.init(seed=1)
    X, y = torch.randn(24, 12) * 3, torch.randint(0, 5, (24,))
    dp = HostDPSGD(clip=0.3, noise=0.8, seed=77, step=10)
    lr = 0.1
    got, _, n = model.train_pass(w, X, y, lr, batch=8, dpsgd=dp)
    want = w.double()
    for i in range(3):
        want = want - lr * _brute(model, want.float(), X[8 * i:8 * i + 8], y[8 * i:8 * i + 8], 0.3, 0.8, 77, 10 + i)
    assert dp.step == 13 and n == 24
    assert float((got.double() - want).abs().max()) < 1e-5


def test_host_non_finite_example_is_dropped():
    model = HostModel("softmax", 3, 2)
    w = model.init(seed=1)
    X = torch.tensor([[1.0, 2.0, 3.0], [float("nan"), 0.0, 0.0]])
    g = model.dpsgd_grad(w, X, torch.tensor([0, 1]), HostDPSGD(clip=1e9, noise=0.0, seed=0))
    ref = _brute(model, w, X[:1], torch.tensor([0]), 1e9, 0.0, 0, 0) / 2
    assert torch.isfinite(g).all() and float((g.double() - ref).abs().max()) < 1e-6


# ------------------------------------------------------------------ the fp32 clip-factor spec
def test_clip_factor_spec():
    sq = np.array([[4.0, 100.0, np.inf, 1e-4]], F32)
    ab = np.array([[1.0, 1.0, 1.0, np.nan]], F32)
    c = D.clip_factors(sq, ab, 2, 1e30)
    assert c.tolist() == [1.0, 1.0, 0.0, 0.0]                    # above every bound: exactly 1; non-finite: 0
    c = D.clip_factors(sq, ab, 2, 1.0)
    bound = (F32(F32(2.0 * 2) * D.ONE_PLUS_GAMMA) + F32(F32(1.0 * 2) * D.U_PLUS_GAMMA))
    assert c[0] == F32(F32(1.0) / bound) and c[0] < F32(0.25)   # the slack makes c smaller than C / (B ||v||)


def _realised(dz, x, c):
    """||bf16(c dz) (x, 1)^T||, the exact norm of a one-row site's realised weight-and-bias contribution."""
    s = torch.from_numpy((dz * c).astype(F32)).to(torch.bfloat16).double()
    return float(s.norm() * math.sqrt(float((x.astype(np.float64) ** 2).sum()) + 1.0))


def test_certified_bound_holds_where_the_computed_norm_alone_does_not():
    """One example, one site: c from the certified bound keeps the realised (bf16-rounded) contribution
    within C for every fixture; c = C / ||v|| on the computed norm (the modelled mistake) exceeds it."""
    rng = np.random.default_rng(3)
    over = 0
    for _ in range(200):
        dz = torch.from_numpy(rng.standard_normal(64).astype(F32)).to(torch.bfloat16).float().numpy()
        x = torch.from_numpy(rng.standard_normal(32).astype(F32)).to(torch.bfloat16).float().numpy()
        ra, rb = F32((dz.astype(np.float64) ** 2).sum()), F32((x.astype(np.float64) ** 2).sum() + 1)
        sq, ab = F32(ra * rb), F32(F32(np.sqrt(ra)) * F32(np.sqrt(rb)))
        clip = F32(0.5 * math.sqrt(float(sq)))
        c = D.clip_factors(np.array([[sq]]), np.array([[ab]]), 1, clip)[0]
        assert _realised(dz, x, c) <= clip
        naive = F32(clip / F32(np.sqrt(sq)))
        over += _realised(dz, x, naive) > clip
    assert over > 0


# ------------------------------------------------------------------ modelled mistakes
def test_mistakes_fail_the_fixtures():
    torch.manual_seed(1)
    model = HostModel("mlp", 6, 3, hidden=8)
    w = model.init(seed=2)
    X, y = torch.randn(4, 6) * 4, torch.randint(0, 3, (4,))
    clip = 0.2
    good = _brute(model, w, X, y, clip, 0.0, 0, 0)
    got = model.dpsgd_grad(w, X, y, HostDPSGD(clip=clip, noise=0.0, seed=0))
    assert float((got.double() - good).abs().max()) < 1e-6
    # per-layer instead of per-example clipping
    w64, gs = w.double(), []
    for n in range(4):
        wn = w64.clone().requires_grad_(True)
        p = model.spec.views(wn)
        h = torch.relu(X[n:n + 1].double() @ p["w1"].t() + p["b1"])
        gs.append(torch.autograd.grad(torch.nn.functional.cross_entropy(h @ p["w2"].t() + p["b2"],
                                                                        y[n:n + 1].long()), wn)[0])
    per_layer = torch.zeros_like(w64)
    for g in gs:
        for e in model.spec.entries:
            part = g[e.offset:e.offset + e.numel]
            per_layer[e.offset:e.offset + e.numel] += part * min(1.0, clip / float(part.norm()))
    assert float((per_layer / 4 - good).abs().max()) > 1e-3
    # the bias term missing from the norm: an example whose features are all zero has only bias
    # gradients, so a clip on the weight part alone would leave it unclipped
    soft = HostModel("softmax", 6, 3)
    w0 = soft.init(seed=4)
    X0, y0 = torch.zeros(2, 6), torch.tensor([0, 2])
    clipped = soft.dpsgd_grad(w0, X0, y0, HostDPSGD(clip=0.05, noise=0.0, seed=0))
    unclipped = soft.dpsgd_grad(w0, X0, y0, HostDPSGD(clip=1e9, noise=0.0, seed=0))
    assert float(unclipped.norm()) > 0.05 and float(clipped.norm()) <= 0.05 * (1 + 1e-6)
    # noise scaled by 1 / M (rows) instead of 1 / B (examples): a 4 x 128-token step
    step = D.DPSGDStep(_spec(), 4, 1.0, 1.0, 0, torch.zeros(1, dtype=torch.int32), "cpu")
    assert step.sigma == float(D.noise_sigma(1.0, 1.0, 4)) == 0.25 != 1.0 / (4 * 128)
    # noise not keyed by the step: consecutive steps must draw fresh noise
    a = HostDPSGD(clip=clip, noise=1.0, seed=5)
    g0 = model.dpsgd_grad(w, X, y, a)
    g1 = model.dpsgd_grad(w, X, y, a)
    assert a.step == 2 and float((g0 - g1).abs().max()) > 1e-3


def _spec():
    from bflc_demo_b200.models.flat import ParamSpec
    return ParamSpec([("a", (8, 768)), ("b", (768, 8))])


# ------------------------------------------------------------------ ptxas
def test_dpsgd_kernels_ptxas_clean(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(nvcc).exists():
        pytest.skip("nvcc not found")
    src = Path(build.CSRC) / "kernels" / "dpsgd_kernels.cu"
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, "-I", str(Path(build.CSRC) / "include"), "-c", str(src),
           "-o", str(tmp_path / "d.o")]
    out = subprocess.run(cmd, capture_output=True, text=True, check=True)
    log = out.stdout + out.stderr
    entries = re.findall(r"Compiling entry function '(\w+)'", log)
    for k in ("k_pe_norm", "k_pe_rows", "k_dpsgd_clip", "k_scale_rows", "k_colsum_fixed", "k_dpsgd_noise"):
        assert any(k in e for e in entries), (k, entries)
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(props) == len(entries) and all(p == ("0", "0", "0") for p in props), log
    assert "C7518" not in log and "C7520" not in log and "serializ" not in log.lower(), log
