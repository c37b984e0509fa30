"""DP-SGD in the persistent MLP trainer, on the host: the opt-in and its refusals (config, CLI, engine), a
numpy model of one fused DP-SGD step (per-row sq / ab of the two R = 1 sites, ``clip_factors``, the scaled
bf16 rows, the fixed-order bias sums, the noise of ``oracle.dp_gauss`` and FedProx after it) against fp64
per-example autograd of the MLP, modelled mistakes that the fixtures must catch, and the DP entry's ptxas
report (no serialized wgmma, spill ceilings)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from bflc_demo_b200 import build
from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.ops.dpsgd import clip_factors, noise_sigma
from bflc_demo_b200.protocol import oracle as O

F32 = np.float32


# ------------------------------------------------------------------ config and CLI
def test_config_accepts_the_opt_in():
    for dtype in ("bf16", "fp8"):
        c = FLConfig(dpsgd_clip=1.0, dpsgd_noise=0.5, dpsgd_fused=True, dtype=dtype).validate()
        assert c.dpsgd_on and c.dpsgd_fused
    assert not FLConfig().validate().dpsgd_fused
    # checkpoints record the config as JSON, the opt-in with it
    c = FLConfig(dpsgd_clip=1.0, dpsgd_fused=True)
    assert FLConfig.from_json(c.to_json()).dpsgd_fused


@pytest.mark.parametrize("kw, why", [
    (dict(), "dpsgd_fused needs dpsgd_clip > 0"),
    (dict(dpsgd_clip=1.0, model="lenet5", dpsgd_conv=True), "applies to the mlp"),
    (dict(dpsgd_clip=1.0, dpsgd_sampling="poisson", samples_per_client=4096), "Poisson sampling needs the generic engine"),
    (dict(dpsgd_clip=1.0, lora_rank=4), "excludes"),
    (dict(dpsgd_clip=1.0, fused_step=False), "fused_step and hidden == 256"),
    (dict(dpsgd_clip=1.0, hidden=128), "fused_step and hidden == 256"),
])
def test_config_refuses(kw, why):
    with pytest.raises(ValueError, match=why):
        FLConfig(dpsgd_fused=True, **kw).validate()


def test_fp8_refusal_stays_without_the_opt_in():
    with pytest.raises(ValueError, match="dtype fp8 is not supported"):
        FLConfig(dpsgd_clip=1.0, dtype="fp8").validate()


@pytest.mark.parametrize("argv, why", [
    (["--model", "mlp", "--dpsgd-fused"], "--dpsgd-fused needs --dpsgd-clip"),
    (["--model", "mlp", "--generic", "--dpsgd-clip", "1", "--dpsgd-fused"], "excludes --generic"),
    (["--model", "lenet5", "--dpsgd-clip", "1", "--dpsgd-fused"], "applies to --model mlp"),
    (["--model", "mlp", "--dpsgd-clip", "1", "--dpsgd-fused", "--dpsgd-sampling", "poisson"],
     "Poisson sampling needs the generic engine"),
    (["--model", "mlp", "--dpsgd-clip", "1"], "fused MLP trainer has no per-example clipping"),
])
def test_cli_refuses(argv, why, capsys):
    from bflc_demo_b200.run import main
    with pytest.raises(SystemExit) as e:
        main(argv)
    assert e.value.code == 2
    assert why in capsys.readouterr().err


def test_cli_accepts_and_picks_the_fused_engine(monkeypatch):
    """--dpsgd-fused passes the CLI checks and reaches FusedEngine (stopped there: no GPU here)."""
    import bflc_demo_b200.engine.fused as fused
    from bflc_demo_b200 import run

    class Stop(Exception):
        pass

    seen = {}

    def fake(cfg, shard, **kw):
        seen["cfg"] = cfg
        raise Stop

    monkeypatch.setattr(fused, "FusedEngine", fake)
    monkeypatch.setattr(torch.cuda, "set_device", lambda *a: None)
    for dtype in ("bf16", "fp8"):
        with pytest.raises(Stop):
            run.main(["--model", "mlp", "--dpsgd-clip", "1", "--dpsgd-noise", "0.8", "--dpsgd-fused", "--dtype", dtype,
                      "--rounds", "1"])
        assert seen["cfg"].dpsgd_fused and seen["cfg"].dtype == dtype


def test_engine_keeps_its_refusal_without_the_opt_in():
    from bflc_demo_b200.engine.fused import FusedEngine
    with pytest.raises(ValueError, match="DP-SGD"):
        FusedEngine(FLConfig.for_world(1, dpsgd_clip=1.0), None)


# ------------------------------------------------------------------ the numpy model of one step
def bf16(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=F32)).to(torch.bfloat16).float().numpy()


class Layout:
    """The flat parameter layout of mlp_spec: w1 [H, D] | b1 [H] | w2 [NC, H] | b2 [NC], 8-aligned."""

    def __init__(self, D, H, NC):
        from bflc_demo_b200.models.mlp import mlp_spec
        self.spec = mlp_spec(D, H, NC)
        self.P = self.spec.total

        self.pad = np.ones(self.P, bool)       # the padding between tensors: no gradient, no noise
        for e in self.spec.entries:
            self.pad[e.offset:e.offset + e.numel] = False

    def flat(self, parts):
        g = np.zeros(self.P, F32)
        for e in self.spec.entries:
            g[e.offset:e.offset + e.numel] = parts[e.name].reshape(-1)
        return g


def fixed_colsum(rows, n_tiles, slots=None):
    """The trainer's bias sums: per 64-row tile two 32-row groups, rows r = k (mod 4) of a group summed in
    order into t[k], the group (t0 + t1) + (t2 + t3); then the groups added to 0 in tile order.  ``slots``
    (a modelled mistake): sum only the first that many groups."""
    B, cols = rows.shape
    pad = np.zeros((n_tiles * 64, cols), F32)
    pad[:B] = rows
    g = np.zeros(cols, F32)
    for p in range(2 * n_tiles if slots is None else slots):
        t = [np.zeros(cols, F32) for _ in range(4)]
        for rr in range(32):
            t[rr & 3] = (t[rr & 3] + pad[32 * p + rr]).astype(F32)
        g = (g + ((t[0] + t[1]).astype(F32) + (t[2] + t[3]).astype(F32)).astype(F32)).astype(F32)
    return g


def fused_step(x, h, dz, dh, lay, clip, noise=0.0, seed=0, word=0, prox=None, mutant=None):
    """One fused DP-SGD step's released gradient from the step's bf16 rows (x [B, D], h [B, H], dz [B, NC]
    with the 1 / B of the mean loss, dh [B, H] relu-masked), as the trainer forms it.  ``prox`` = (mu, w, w0)
    adds the proximal term after the noise.  ``mutant`` names a modelled mistake."""
    B, D = x.shape
    sq2 = lambda a: np.sum(a.astype(np.float64) ** 2, 1).astype(F32)
    dzn = dz
    if mutant == "last_class_dropped":
        dzn = dz[:, :-1]
    elif mutant == "junk_pad_class":        # a padding column of the 64-wide tile read as a class
        dzn = np.concatenate([dz, np.abs(dz).max(1, keepdims=True)], 1)
    a0, hb = sq2(dzn), sq2(h)
    a1 = sq2(dh[:, :dh.shape[1] // 4]) if mutant == "own_slice_dh" else sq2(dh)
    xb = sq2(x[:, :D // 64 * 64]) if mutant == "k_tail_dropped" else sq2(x)
    one = F32(0) if mutant == "no_bias_one" else F32(1)
    with np.errstate(all="ignore"):
        b0, b1 = (hb + one).astype(F32), (xb + one).astype(F32)
        sq = np.stack([(a0 * b0).astype(F32), (a1 * b1).astype(F32)])
        ab = np.stack([(np.sqrt(a0) * np.sqrt(b0)).astype(F32), (np.sqrt(a1) * np.sqrt(b1)).astype(F32)])
    if mutant == "site_omitted":
        sq, ab = sq[:1], ab[:1]
    c = clip_factors(sq, ab, B, clip)
    zero = c == 0
    with np.errstate(all="ignore"):
        if mutant == "clip_after_rounding":
            dzs, dhs = (dz * c[:, None]).astype(F32), (dh * c[:, None]).astype(F32)
        elif mutant == "unscaled_rows":
            dzs, dhs = dz.copy(), dh.copy()
        else:
            dzs, dhs = bf16(dz * c[:, None]), bf16(dh * c[:, None])
        dzs[zero], dhs[zero] = 0, 0
        hm = h.copy()
        if mutant != "dropped_h_kept":
            hm[zero] = 0
        n_tiles = -(-B // 64)
        parts = {"w1": (dhs.astype(np.float64).T @ x.astype(np.float64)).astype(F32),
                 "w2": (dzs.astype(np.float64).T @ hm.astype(np.float64)).astype(F32),
                 "b1": fixed_colsum(dhs, n_tiles, n_tiles if mutant == "half_bias_slots" else None),
                 "b2": fixed_colsum(dzs, n_tiles, n_tiles if mutant == "half_bias_slots" else None)}
    g = lay.flat(parts)
    sigma = noise_sigma(noise, clip, B)

    def add_noise(g):
        if sigma == 0:
            return g
        if mutant == "tile_local_noise":   # each tensor keyed from its own index 0
            xi = np.zeros(lay.P, F32)
            for e in lay.spec.entries:
                xi[e.offset:e.offset + e.numel] = O.dp_gauss(seed, word, 0, e.numel, O.DPSGD_SITE)
        else:
            xi = O.dp_gauss(seed, word, 0, lay.P, O.DPSGD_SITE)
        if mutant != "noise_in_padding":
            xi = np.where(lay.pad, F32(0), xi).astype(F32)
        return (g + (sigma * xi).astype(F32)).astype(F32)

    def add_prox(g):
        mu, w, w0 = prox
        return (np.float64(mu) * (w - w0).astype(F32).astype(np.float64) + g.astype(np.float64)).astype(F32)

    if prox is not None and mutant == "noise_after_prox":
        g = add_noise(add_prox(g))
    else:
        g = add_noise(g)
        if prox is not None:
            g = add_prox(g)
    return dict(sq=sq, ab=ab, c=c, dz=dzs, dh=dhs, h=hm, g=g)


MUTANTS = ["site_omitted", "no_bias_one", "own_slice_dh", "clip_after_rounding", "tile_local_noise",
           "noise_after_prox", "dropped_h_kept"]


def make_case(B=40, D=48, H=32, NC=10, seed=0, blow_up=None):
    """Seeded MLP and batch; the rows the trainer would store (bf16) and the fp64 per-example gradients
    of the mean loss by autograd.  ``blow_up``: an example whose h row is inf."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, D, generator=g).to(torch.bfloat16).double()
    y = torch.randint(0, NC, (B,), generator=g)
    w1 = (torch.rand(H, D, generator=g) * 2 - 1) / D ** 0.5
    b1 = torch.rand(H, generator=g) * 0.1
    w2 = (torch.rand(NC, H, generator=g) * 2 - 1) / H ** 0.5 * 2
    b2 = torch.zeros(NC)
    W = [t.double().requires_grad_(True) for t in (w1, b1, w2, b2)]
    per = []
    for n in range(B):
        hn = torch.relu(x[n:n + 1] @ W[0].t() + W[1])
        ln = torch.nn.functional.cross_entropy(hn @ W[2].t() + W[3], y[n:n + 1]) / B
        per.append(torch.cat([t.reshape(-1) for t in torch.autograd.grad(ln, W)]).detach().numpy())
    with torch.no_grad():
        h = torch.relu(x @ W[0].t() + W[1])
        p = torch.softmax(h @ W[2].t() + W[3], 1)
        dz = (p - torch.nn.functional.one_hot(y, NC).double()) / B
        dh = (dz @ W[2]) * (h > 0)
    rows = [bf16(t.numpy()) for t in (x, h, dz, dh)]
    if blow_up is not None:
        rows[1][blow_up] = np.inf
    return rows, np.array(per), Layout(D, H, NC), [t.detach().numpy() for t in W]


def per_example_flat(per, lay, shapes=None):
    """autograd's per-example gradients [B, w1 | b1 | w2 | b2] in the flat layout."""
    out = np.zeros((per.shape[0], lay.P))
    o = 0
    for e in lay.spec.entries:
        out[:, e.offset:e.offset + e.numel] = per[:, o:o + e.numel]
        o += e.numel
    return out


def fixtures(mutant=None):
    """The checks a fused DP-SGD step must pass; a mistake fails at least one of them (returns False)."""
    (x, h, dz, dh), per, lay, W = make_case()
    B = x.shape[0]
    G = per_example_flat(per, lay)
    norm2 = (G ** 2).sum(1)
    clip = float(np.median(np.sqrt(norm2)) * B)
    r = fused_step(x, h, dz, dh, lay, clip, mutant=mutant)
    ok = True
    # F1: the two sites' sq sum to each example's squared gradient norm (bf16 rows: 2^-6 relative)
    ok &= bool(np.allclose(r["sq"].sum(0), norm2, rtol=2.0 ** -6))
    # F2: the released rows are bf16(row * c), k_scale_rows' rule
    ok &= bool(np.array_equal(r["dz"], bf16(dz * r["c"][:, None])) and np.array_equal(r["dh"], bf16(dh * r["c"][:, None])))
    # F3: the release is the fp64 sum of c_n g_n within the rows' bf16 rounding, each example at most C / B
    ref = (r["c"][:, None].astype(np.float64) * G).sum(0)
    mag = (r["c"][:, None].astype(np.float64) * np.abs(G)).sum(0)
    ok &= bool(np.all(np.abs(r["g"] - ref) <= 2.0 ** -7 * mag + 1e-12))
    ok &= bool(np.all(r["c"] * np.sqrt(norm2) <= clip / B * (1 + 1e-6)))
    # F4: the noise is oracle.dp_gauss over the flat index, then FedProx
    seed, word, z, mu = 0xABCDEF, 17, 1.3, F32(0.25)
    w = np.random.default_rng(1).standard_normal(lay.P).astype(F32)
    w0 = (w * F32(0.5)).astype(F32)
    rn = fused_step(x, h, dz, dh, lay, clip, z, seed, word, prox=(mu, w, w0), mutant=mutant)
    xi = np.where(lay.pad, F32(0), O.dp_gauss(seed, word, 0, lay.P, O.DPSGD_SITE)).astype(F32)
    sig = noise_sigma(z, clip, B)
    want = (r["g"] + (sig * xi).astype(F32)).astype(F32)
    want = (np.float64(mu) * (w - w0).astype(F32).astype(np.float64) + want.astype(np.float64)).astype(F32)
    ok &= bool(np.array_equal(rn["g"], want))
    # F5: an example whose h is inf is dropped; its rows release exact zeros and the step is finite
    (x2, h2, dz2, dh2), _, _, _ = make_case(blow_up=5)
    with np.errstate(all="ignore"):
        dz2[5] = np.nan
        dh2[5] = np.nan
    rd = fused_step(x2, h2, dz2, dh2, lay, clip, mutant=mutant)
    ok &= bool(rd["c"][5] == 0 and np.all(np.isfinite(rd["g"])))
    keep = np.arange(B) != 5
    ok &= bool(np.all(rd["c"][keep] > 0))
    return ok


def test_model_passes_every_fixture():
    assert fixtures()


@pytest.mark.parametrize("mutant", MUTANTS)
def test_every_modelled_mistake_fails_a_fixture(mutant):
    assert not fixtures(mutant)


def test_model_against_fp64_per_example_autograd():
    """With C above every bound the release is the plain mean-loss gradient; with a binding C each example is
    scaled to at most C / B and the release is the fp64 sum of the scaled per-example gradients."""
    (x, h, dz, dh), per, lay, _ = make_case(seed=3)
    B = x.shape[0]
    G = per_example_flat(per, lay)
    r = fused_step(x, h, dz, dh, lay, 1e30)
    assert np.all(r["c"] == 1)
    assert np.allclose(r["g"], G.sum(0), rtol=2.0 ** -6, atol=2.0 ** -7 * np.abs(G).sum(0).max())
    norms = np.sqrt((G ** 2).sum(1))
    clip = float(norms.min() * B * 0.5)       # every example clipped
    r = fused_step(x, h, dz, dh, lay, clip)
    assert np.all(r["c"] < 1)
    assert np.all(r["c"] * norms <= clip / B * (1 + 1e-6))
    assert np.all(r["c"] * norms >= clip / B * 0.97)   # the bound is tight to the bf16 rounding slack


# ------------------------------------------------------------------ the DP entry's ptxas report
SRC = build.CSRC / "kernels" / "mlp_round_sm100.cu"
# instantiation -> (spill store bytes, spill load bytes) ceilings of mlp_dpsgd_round_kernel
DP_SPILL_CEILING = {"ILb0E": (716, 1340),   # bf16
                    "ILb1E": (756, 1304)}   # fp8


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("no nvcc")
    out = tmp_path_factory.mktemp("ptxas") / "m.o"
    inc = [f"-I{build.CSRC / d}" for d in ("include", "ledger", "runtime")]
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, *inc, "-c", str(SRC), "-o", str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    log = proc.stdout + proc.stderr
    assert proc.returncode == 0, log[-3000:]
    return log


def test_dp_entry_wgmma_not_serialized(ptxas_log):
    entries = re.findall(r"Compiling entry function '(\w*mlp_dpsgd_round_kernel\w*)'", ptxas_log)
    assert len(entries) == 2, ptxas_log[-3000:]
    serialized = [ln for ln in ptxas_log.splitlines()
                  if re.search(r"\(C75(18|20)\)", ln) and "mlp_dpsgd_round_kernel" in ln]
    assert not serialized, "\n".join(serialized)


def test_dp_entry_spills_do_not_grow(ptxas_log):
    props = re.findall(r"Function properties for (\w*mlp_dpsgd_round_kernel(ILb[01]E)\w*)\s*\n\s*"
                       r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ptxas_log)
    found = {inst: (int(st), int(ld)) for _, inst, _, st, ld in props}
    assert set(found) == set(DP_SPILL_CEILING), ptxas_log[-3000:]
    for inst, (st, ld) in found.items():
        cs, cl = DP_SPILL_CEILING[inst]
        assert st <= cs and ld <= cl, f"{inst}: {st} B spill stores / {ld} B loads, ceiling {cs} / {cl}"


# ------------------------------------------------------------------ shape mistakes and their GPU checks
# (B, in_dim, C) of the GPU conformance matrix (hidden 256)
SHAPES = [(32, 784, 62), (200, 784, 62), (512, 784, 62), (256, 784, 57), (256, 784, 64), (256, 64, 62),
          (256, 512, 62)]


def matrix_rows(B, D, C, H=256, seed=0, drop=None):
    """bf16 rows of one step as the trainer stores them: x nonzero in every K-block (the tail included),
    half the rows labelled C - 1 (the largest |dz| of those rows sits in the last class); ``drop``: an
    example whose h is inf."""
    rng = np.random.default_rng(seed + B + D + C)
    x = bf16(rng.random((B, D)) ** 2)
    w1 = rng.standard_normal((H, D)) / D ** 0.5
    w2 = rng.standard_normal((C, H)) / H ** 0.5 * 2
    y = rng.integers(0, C, B)
    y[1::2] = C - 1
    h = np.maximum(x.astype(np.float64) @ w1.T + 0.05, 0)
    z = h @ w2.T
    p = np.exp(z - z.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    dz = (p - np.eye(C)[y]) / B
    dh = (dz @ w2) * (h > 0)
    rows = [bf16(t) for t in (x, h, dz, dh)]
    if drop is not None:
        rows[1][drop] = np.inf
    return rows


SHAPE_MUTANTS = {"k_tail_dropped": "norms", "last_class_dropped": "norms", "junk_pad_class": "norms",
                 "unscaled_rows": "stored_rows", "dropped_h_kept": "stored_rows", "half_bias_slots": "release",
                 "noise_in_padding": "padding"}


def run_helper(helper, B, D, C, mutant=None):
    """One GPU check of test_gpu_dpsgd_trainer_conformance on the numpy model's step (with ``mutant``)."""
    import test_gpu_dpsgd_trainer_conformance as G
    x, h, dz, dh = matrix_rows(B, D, C, drop=B // 2)
    lay = Layout(D, 256, C)
    with np.errstate(all="ignore"):
        ref = fused_step(x, h, dz, dh, lay, 1e30)
        clip = float(np.median(np.sqrt(ref["sq"].astype(np.float64).sum(0)[np.isfinite(ref["sq"].sum(0))])) * B)
        r = fused_step(x, h, dz, dh, lay, clip, mutant=mutant)
    live = np.isfinite(ref["sq"].sum(0))
    if helper == "norms":
        G.check_norms(r["sq"][:, live], r["ab"][:, live], x[live], h[live], dz[live], dh[live])
    elif helper == "stored_rows":
        assert 0.2 < float((r["c"][live] < 1).mean()) < 0.8 and r["c"][B // 2] == 0
        G.check_stored_rows(r["c"], (h, dz, dh), (r["h"], r["dz"], r["dh"]))
        G.check_certified_bound(x, r["h"], r["dz"], r["dh"], clip)
    elif helper == "release":
        G.check_release(r["g"], x, r["h"], r["dz"], r["dh"], lay.spec)
    else:
        rn = fused_step(x, h, dz, dh, lay, clip, 1.3, 0xABC, 5, mutant=mutant)
        G.check_padding(rn["g"], lay.spec, "noised release")


@pytest.mark.parametrize("B, D, C", SHAPES, ids=[f"B{b}-{d}x256x{c}" for b, d, c in SHAPES])
def test_model_passes_every_gpu_check(B, D, C):
    for helper in ("norms", "stored_rows", "release", "padding"):
        run_helper(helper, B, D, C)


@pytest.mark.parametrize("mutant", sorted(SHAPE_MUTANTS))
@pytest.mark.parametrize("B, D, C", SHAPES, ids=[f"B{b}-{d}x256x{c}" for b, d, c in SHAPES])
def test_every_shape_mistake_fails_its_gpu_check(B, D, C, mutant):
    if mutant == "k_tail_dropped" and D % 64 == 0:
        pytest.skip("no partial K-block at this in_dim")
    if mutant == "noise_in_padding" and Layout(D, 256, C).pad.sum() == 0:
        pytest.skip("no padding between tensors at this shape")
    if mutant == "half_bias_slots" and B <= 32:
        pytest.skip("one M-tile whose second 32-row slot is empty")
    with pytest.raises(AssertionError):
        run_helper(SHAPE_MUTANTS[mutant], B, D, C, mutant)


# ------------------------------------------------------------------ refusals of the chain's shapes
@pytest.mark.parametrize("C", [2, 10, 56])
@pytest.mark.parametrize("mode", ["dpsgd", "fp8"])
def test_class_counts_outside_the_chain_are_refused_at_construction(C, mode):
    """The chain's tiles are 64 classes wide (ncp == 64): fewer than 57 classes have neither a DP-SGD nor an
    fp8 trainer, and FlatMLP and FusedEngine say so before anything is allocated on a device."""
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec
    spec = mlp_spec(784, 256, C)
    m = torch.zeros(spec.total)
    kw = dict(dpsgd_clip=1.0) if mode == "dpsgd" else dict(fp8=True)
    with pytest.raises(ValueError, match="57..64 classes"):
        FlatMLP(spec, m, m.bfloat16(), torch.zeros_like(m), 256, **kw)
    ckw = dict(dpsgd_clip=0.5, dpsgd_noise=1.0, dpsgd_fused=True) if mode == "dpsgd" else dict(dtype="fp8")
    cfg = FLConfig.for_world(1, model="mlp", hidden=256, batch_size=256, samples_per_client=1024,
                             learning_rate=0.05, **ckw)
    with pytest.raises(ValueError, match="57..64 classes"):
        FusedEngine(cfg, femnist_like(1, 1024, seed=7, n_classes=C, only=0)[0])
