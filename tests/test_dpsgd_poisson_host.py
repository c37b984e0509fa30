"""Poisson-sampled DP-SGD on the CPU: the sampled Gaussian accountant against numerical integration of the Renyi
divergence, the capacity against scipy's binomial tail, the oracle sampler, the clip-factor mirror with padding,
the config and CLI refusals, and a host-simulator run (protocol/privacy.py, protocol/oracle.py, host/)."""
import math

import numpy as np
import pytest

from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.ops.dpsgd import clip_factors
from bflc_demo_b200.protocol import privacy as P
from bflc_demo_b200.protocol.oracle import poisson_sample, poisson_threshold

try:
    from scipy import integrate, stats
except ImportError:          # only the scipy cross-checks need it
    integrate = stats = None

needs_scipy = pytest.mark.skipif(stats is None, reason="scipy not installed")


# ------------------------------------------------------------------ accountant
def _rdp_quad(q, z, alpha, reverse):
    """D_alpha(mu || nu) by quadrature, mu = (1 - q) N(0, z^2) + q N(1, z^2), nu = N(0, z^2) (reverse: D(nu || mu)),
    written as log1p of the integral of nu (rho^alpha - 1) (reverse: mu (rho^-alpha - 1)), rho = mu / nu, so that
    small divergences keep their digits."""
    def log_rho(x):
        return math.log1p(q * math.expm1((2 * x - 1) / (2 * z * z)))

    def f(x):
        lr = log_rho(x)
        e = (1 - alpha) * lr if reverse else alpha * lr         # log of mu^alpha nu^-alpha (reverse: nu mu ...)
        lp = stats.norm.logpdf(x, 0, z)
        # nu e^e - (reverse: mu) nu^... written so that a small e keeps its digits and a large one cannot overflow
        base = math.exp(lp + lr) if reverse else math.exp(lp)
        return math.exp(lp) * math.expm1(e) + (math.exp(lp) - base) if e < 1 else math.exp(lp + e) - base

    lo, hi = -12 * z - 2, alpha + 12 * z + 2      # the tilted mass sits near x = alpha
    val, _ = integrate.quad(f, lo, hi, limit=1000, epsabs=0, epsrel=1e-10, points=[0.5, alpha / 2])
    return math.log1p(val) / (alpha - 1)


@needs_scipy
@pytest.mark.parametrize("q, z, alpha", [(1e-3, 1.0, 2), (1e-3, 0.8, 32), (0.01, 1.0, 8), (0.05, 2.0, 16),
                                         (0.2, 1.5, 5), (0.5, 3.0, 12), (0.5, 1.0, 3)])
def test_sampled_gaussian_rdp_against_quadrature_in_both_orders(q, z, alpha):
    got = P.sampled_gaussian_rdp(q, z, alpha)
    fwd = _rdp_quad(q, z, alpha, False)
    rev = _rdp_quad(q, z, alpha, True)
    # the binomial expansion is D(mixture || base); for integer alpha the reverse order is no larger
    # (Mironov et al. 2019, Thm 5), so the expansion bounds both
    assert got == pytest.approx(fwd, rel=1e-6, abs=1e-12)
    assert rev <= got * (1 + 1e-6) + 1e-12


@pytest.mark.parametrize("z, alpha", [(1.0, 2), (0.7, 10), (2.5, 256)])
def test_rdp_at_q_one_is_the_gaussian(z, alpha):
    assert P.sampled_gaussian_rdp(1.0, z, alpha) == alpha / (2 * z * z)


def test_epsilon_is_monotone_in_q_and_steps_and_below_the_partition_accountant():
    from bflc_demo_b200.engine.generic import dpsgd_epsilon
    qs = [1e-3, 4e-3, 1e-2, 5e-2]
    eps_q = [P.poisson_epsilon(q, 1.0, 500, 1e-5) for q in qs]
    assert all(a < b for a, b in zip(eps_q, eps_q[1:]))
    eps_t = [P.poisson_epsilon(0.01, 1.0, t, 1e-5) for t in (1, 10, 100, 1000)]
    assert all(a < b for a, b in zip(eps_t, eps_t[1:]))
    # the README's 2-layer GPT command: B 16 of S 2048, 128 steps a round, z 1, delta 1e-5
    cfg = FLConfig(model="gpt", lora_rank=8, batch_size=16, dpsgd_clip=1.0, dpsgd_noise=1.0)
    q = poisson_threshold(16, 2048) / 2.0 ** 32
    for rounds, want in ((1, 1.13), (10, 1.85)):
        poisson = P.poisson_epsilon(q, 1.0, 128 * rounds, 1e-5)
        assert poisson == pytest.approx(want, abs=0.01)
        assert poisson < dpsgd_epsilon(cfg, 128 * rounds, 2048 // 16)[0]
    assert P.poisson_epsilon(q, 1.0, 0, 1e-5) == 0.0 and P.poisson_epsilon(q, 0.0, 5, 1e-5) == math.inf


def test_rdp_conversion_is_balle_et_al():
    rdp, a, d = 0.3, 7, 1e-6
    assert P.rdp_to_epsilon(rdp, a, d) == pytest.approx(rdp + math.log(6 / 7) - (math.log(d) + math.log(7)) / 6)


# ------------------------------------------------------------------ capacity
@needs_scipy
@pytest.mark.parametrize("S, B", [(4096, 512), (2048, 16), (60000, 512), (100, 50), (64, 63), (10, 1), (17, 9)])
def test_capacity_against_scipy(S, B):
    q = poisson_threshold(B, S) / 2.0 ** 32
    cap = P.poisson_capacity(S, q)
    assert cap <= S and (cap % 8 == 0 or cap == S)
    if cap < S:
        assert stats.binom.sf(cap, S, q) <= P.POISSON_ETA * (1 + 1e-6)
        assert P.binomial_tail(S, q, cap) == pytest.approx(stats.binom.sf(cap, S, q), rel=1e-6)
    if cap >= 8:
        assert stats.binom.sf(cap - 8, S, q) > P.POISSON_ETA
    assert P.binomial_tail(S, q, S) == 0.0


def test_capacity_of_the_documented_configurations():
    assert P.poisson_capacity(4096, poisson_threshold(512, 4096) / 2 ** 32) == 672
    assert P.poisson_capacity(2048, poisson_threshold(16, 2048) / 2 ** 32) == 56
    assert P.poisson_capacity(64, poisson_threshold(63, 64) / 2 ** 32) == 64      # cap = S: no overflow


# ------------------------------------------------------------------ oracle sampler
def test_sampler_is_deterministic_and_keyed_by_seed_and_step():
    thr = poisson_threshold(64, 1000)
    a = poisson_sample(1, 5, 1000, thr, 200)
    assert np.array_equal(a[0], poisson_sample(1, 5, 1000, thr, 200)[0])
    assert not np.array_equal(a[0], poisson_sample(2, 5, 1000, thr, 200)[0])
    assert not np.array_equal(a[0], poisson_sample(1, 6, 1000, thr, 200)[0])
    idx, count, over = a
    assert not over and np.all(np.diff(idx[:count]) > 0) and np.all(idx[count:] == 0)


def test_sample_counts_have_mean_q_s():
    S, B, n = 500, 20, 10_000
    thr = poisson_threshold(B, S)
    q = thr / 2 ** 32
    counts = np.array([poisson_sample(77, t, S, thr, S)[1] for t in range(n)])
    se = math.sqrt(S * q * (1 - q) / n)
    assert abs(counts.mean() - q * S) < 5 * se


def test_truncation_keeps_the_first_cap_in_record_order():
    thr = poisson_threshold(900, 1000)
    full, n, _ = poisson_sample(3, 0, 1000, thr, 1000)
    idx, count, over = poisson_sample(3, 0, 1000, thr, 40)
    assert over and count == 40 and np.array_equal(idx, full[:40]) and n > 40


def test_threshold_rounding_is_exact_at_its_edges():
    assert poisson_threshold(1, 2) == 1 << 31
    assert poisson_threshold(1, 3) == (1 << 32) // 3
    assert poisson_threshold(2 ** 24 - 1, 2 ** 24) == (1 << 32) - 256
    assert poisson_threshold(1, 2 ** 24) == 256
    # floor: thr / 2^32 <= q < (thr + 1) / 2^32
    for B, S in ((7, 13), (16, 2048), (512, 60000), (3, 1 << 24)):
        t = poisson_threshold(B, S)
        assert t * S <= B << 32 < (t + 1) * S
    with pytest.raises(ValueError):
        poisson_threshold(5, 5)
    with pytest.raises(ValueError):
        poisson_threshold(0, 5)
    # the compare is u < thr: a record whose uniform is u is out at thr = u and in at thr = u + 1
    from bflc_demo_b200.protocol.oracle import DPSGD_SAMPLE_SITE, philox4x32_10
    S, seed, step = 64, 9, 3
    g = np.arange(S // 4, dtype=np.uint32)
    w = philox4x32_10((g, np.zeros_like(g), np.full(g.shape, step, np.uint32),
                       np.full(g.shape, DPSGD_SAMPLE_SITE, np.uint32)), seed, 0)
    u = np.stack(w, axis=1).reshape(-1)
    for j in (0, 1, 2, 3, 37, 63):
        t = int(u[j])
        if 0 < t < (1 << 32) - 1:
            below = poisson_sample(seed, step, S, t, S)
            above = poisson_sample(seed, step, S, t + 1, S)
            assert j not in below[0][:below[1]] and j in above[0][:above[1]]
            assert set(above[0][:above[1]]) - set(below[0][:below[1]]) == {j}


# ------------------------------------------------------------------ clip factors with padding
def test_clip_factors_with_n_valid():
    rng = np.random.default_rng(0)
    sq = rng.random((3, 10)).astype(np.float32) * 1e-3
    ab = rng.random((2, 10)).astype(np.float32) * 1e-3
    sq[:, 8] = np.inf                       # a padding slot that would be dropped
    full = clip_factors(sq, ab, 4, 0.01)
    got = clip_factors(sq, ab, 4, 0.01, n_valid=6)
    assert np.array_equal(got[:6], full[:6]) and np.all(got[6:] == 0)
    assert np.array_equal(clip_factors(sq, ab, 4, 0.01, n_valid=None), full)
    assert np.all(clip_factors(sq, ab, 4, 0.01, n_valid=0) == 0)


# ------------------------------------------------------------------ config and CLI
def test_config_default_and_refusals():
    assert FLConfig().dpsgd_sampling == "partition"
    FLConfig(dpsgd_clip=1.0, dpsgd_sampling="poisson").validate()
    with pytest.raises(ValueError, match="needs dpsgd_clip"):
        FLConfig(dpsgd_sampling="poisson").validate()
    with pytest.raises(ValueError, match="partition or poisson"):
        FLConfig(dpsgd_clip=1.0, dpsgd_sampling="shuffle").validate()
    assert not FLConfig(dpsgd_sampling="partition").dpsgd_poisson


def test_resolve_seed_exists_for_poisson_without_noise():
    from bflc_demo_b200.engine.generic import resolve_dpsgd_seed
    assert resolve_dpsgd_seed(FLConfig(dpsgd_clip=1.0, dpsgd_seed=3), 0) == 0
    assert resolve_dpsgd_seed(FLConfig(dpsgd_clip=1.0, dpsgd_seed=3, dpsgd_sampling="poisson"), 0) != 0
    assert resolve_dpsgd_seed(FLConfig(dpsgd_clip=1.0, dpsgd_sampling="poisson"), 0) != 0


@pytest.mark.parametrize("argv, msg", [
    (["--dpsgd-sampling", "poisson"], "needs --dpsgd-clip"),
    (["--dpsgd-clip", "1", "--dpsgd-sampling", "poisson"], "needs the generic engine"),
    (["--model", "bert", "--lora-rank", "8", "--packed", "--dpsgd-clip", "1", "--dpsgd-sampling", "poisson"],
     "--packed"),
])
def test_cli_refusals(argv, msg, capsys):
    from bflc_demo_b200 import run
    with pytest.raises(SystemExit) as e:
        run.main(argv)
    assert e.value.code == 2 and msg in capsys.readouterr().err


def test_cli_takes_the_flag(monkeypatch):
    """run.main's own parser: the flag reaches the DP-SGD fields (the run stops right after them), and its
    default is partition."""
    from bflc_demo_b200 import run
    seen = []
    real = run.dpsgd_fields

    class Parsed(Exception):
        pass

    def spy(ap, a):
        seen.append(real(ap, a))
        raise Parsed

    monkeypatch.setattr(run, "dpsgd_fields", spy)
    for argv, want in ((["--generic", "--dpsgd-clip", "1", "--dpsgd-sampling", "poisson"], "poisson"),
                       (["--generic", "--dpsgd-clip", "1"], "partition")):
        with pytest.raises(Parsed):
            run.main(argv)
        assert seen[-1]["dpsgd_sampling"] == want


def test_too_small_shards_are_refused():
    with pytest.raises(ValueError, match="samples_per_client >= 2"):
        FLConfig(dpsgd_clip=1.0, dpsgd_sampling="poisson", batch_size=100, samples_per_client=150).validate()
    FLConfig(dpsgd_clip=1.0, batch_size=100, samples_per_client=100).validate()      # partition: fine
    import torch

    from bflc_demo_b200.host.models import HostDPSGD, HostModel
    model = HostModel("softmax", 5, 2)
    X, y = torch.randn(12, 5), torch.randint(0, 2, (12,))
    with pytest.raises(ValueError, match="more shard rows than the batch"):
        model.train_pass(model.init(seed=1), X, y, 0.1, 8, dpsgd=HostDPSGD(1.0, 0.0, 3, poisson=True))


# ------------------------------------------------------------------ host simulator
def test_host_sim_poisson_runs_with_a_consistent_ledger():
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.host import sim
    from bflc_demo_b200.host.models import HostModel
    cfg = FLConfig.for_world(6, learning_rate=0.05, batch_size=50, dpsgd_clip=1.0, dpsgd_noise=1.0, dpsgd_seed=4,
                             dpsgd_sampling="poisson")
    shards = femnist_like(6, 300, seed=1)
    test = femnist_like(1, 200, seed=1, only=0)[0]
    model = HostModel("mlp", 784, 62, hidden=32, scale_inputs=1 / 255.0)
    led, clients, _, _ = sim.run(cfg, shards, test, model=model, rounds=2, log=None)
    assert led.epoch() >= 2 and led.verify_chain()
    stepped = [c for c in clients if c.dpsgd.step > 0]
    assert stepped and all(c.dpsgd.poisson for c in clients)
    eps, delta = sim.host_poisson_epsilon(cfg, stepped[0])
    assert 0 < eps < math.inf and delta > cfg.dp_delta


def test_host_poisson_pass_against_an_independent_reference():
    """The host pass against per-example autograd written out here: each step's oracle sample, clip_C of each
    example's gradient of softmax regression, summed, plus z C xi, over B (never the count)."""
    import torch

    from bflc_demo_b200.host.models import HostDPSGD, HostModel
    from bflc_demo_b200.protocol.oracle import DPSGD_SITE, dp_gauss
    model = HostModel("softmax", 5, 2)
    g = torch.Generator().manual_seed(0)
    X, y = torch.randn(40, 5, generator=g), torch.randint(0, 2, (40,), generator=g)
    w0 = model.init(seed=1)
    clip, z, seed, B, lr = 0.3, 0.7, 12345, 8, 0.1
    w1, cost, n = model.train_pass(w0, X, y, lr, B, dpsgd=HostDPSGD(clip, z, seed, poisson=True))
    assert n == 40 and math.isfinite(cost)
    W = w0.double().clone()
    thr = poisson_threshold(B, 40)
    cap = P.poisson_capacity(40, thr / 2 ** 32)
    for t in range(5):
        idx, count, _ = poisson_sample(seed, t, 40, thr, cap)
        tot = torch.zeros_like(W)
        for j in idx[:count]:
            wv = W.clone().requires_grad_()
            V = model.spec.views(wv)
            loss = torch.nn.functional.cross_entropy(X[j:j + 1].double() @ V["w"].t() + V["b"], y[j:j + 1].long())
            gj, = torch.autograd.grad(loss, wv)
            tot += gj * min(1.0, clip / float(gj.norm()))
        xi = torch.from_numpy(dp_gauss(seed, t, 0, W.numel(), DPSGD_SITE)).double()
        W = W - lr * (tot + float(np.float32(z) * np.float32(clip)) * xi) / B
    assert torch.allclose(w1.double(), W, rtol=0, atol=1e-5), float((w1.double() - W).abs().max())


# ------------------------------------------------------------------ ptxas
def test_sampler_kernel_has_no_spills_and_no_stack(tmp_path):
    import re
    import shutil
    import subprocess
    from pathlib import Path

    from bflc_demo_b200 import build
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(nvcc).exists():
        pytest.skip("nvcc not found")
    src = Path(build.CSRC) / "kernels" / "dpsgd_kernels.cu"
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, "-I", str(Path(build.CSRC) / "include"), "-c", str(src),
           "-o", str(tmp_path / "d.o")]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    log = proc.stdout + proc.stderr
    assert proc.returncode == 0, log[-3000:]
    m = re.search(r"Function properties for \w*k_dpsgd_poisson_sample\w*\s*\n\s*(\d+) bytes stack frame, (\d+) bytes "
                  r"spill stores, (\d+) bytes spill loads", log)
    assert m, log[-3000:]
    assert m.groups() == ("0", "0", "0"), m.group(0)
