"""Differentially private aggregation on the GPU: k_update_norms and the DP consensus kernels, checked
through the one-GPU replica harness of test_gpu_robust_aggregation.py, the engines in solo mode, a
checkpoint / resume, and (2+ GPUs) the multi-GPU check.

Every round is recomputed with the numpy oracle (protocol/oracle.py ``dp_device_combine``, then
``server_step``) from the previous global model, the selected uploads and the device's own norms, all
read back from the heaps, and compared bit for bit (NaN compared as NaN)."""
from __future__ import annotations

import json
import math
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.protocol.oracle import dp_device_combine, dp_gauss, dp_norm, server_step

sys.path.insert(0, str(Path(__file__).resolve().parent))
from test_gpu_robust_aggregation import COMM, N_VAL, TRAINER, crafted_uploads, same  # noqa: E402
from test_gpu_server_optimizer import ServerOptHarness  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
SEED = 0x0DDC0FFEE


class _DpModule:
    """The native module, with the server optimizer's and DP's arguments added to every consensus launch,
    and every rank's fed_update_norms launched in front of the round's first one (the harness launches
    rank 0's consensus first; every upload is published by then)."""

    def __init__(self, mod, kw: dict, feds, dp_off: int):
        self._mod, self._kw, self._feds, self._off = mod, kw, feds, dp_off

    def __getattr__(self, name):
        return getattr(self._mod, name)

    def fed_consensus_aggregate(self, fed, *a, **kw):
        if fed["rank"] == 0:
            for f in self._feds:
                self._mod.fed_update_norms(f, self._off)
        return self._mod.fed_consensus_aggregate(fed, *a, **kw, **self._kw)


class DpHarness(ServerOptHarness):
    """ReplicaHarness with DP (and optionally a server optimizer): heaps laid out with the dp page, host
    ledgers that expect the DP word in every block record."""

    def __init__(self, R: int, n_params: int, *, clip: float, noise: float = 0.0, server_opt: str = "none", **kw):
        from bflc_demo_b200._native import ledger
        from bflc_demo_b200.parallel.layout import HeapLayout

        super().__init__(R, n_params, server_opt=server_opt, **kw)
        base = self.m._mod
        self.cfg = FLConfig(server_opt=server_opt, dp_clip=clip, dp_noise=noise, dp_seed=SEED,
                            aggregation=self.aggregation, aggregate_count=kw["aggregate_count"],
                            needed_updates=kw["aggregate_count"], trim=self.trim).validate()
        self.clip, self.noise = (float(x) for x in self.cfg.dp_constants)
        self.layout = HeapLayout(n_params, self.layout.ring_slots, server_state=self.cfg.server_state_vectors, dp=True)
        self.heaps = self.ptrs = None
        self.heaps = [base.SymmHeap(self.layout.total_bytes, 0, 1, 0, "local") for _ in range(R)]
        self.ptrs = [h.local_ptr() for h in self.heaps]
        self.feds = [self.layout.fed_dict(r, R, self.ptrs, 0) for r in range(R)]
        kwargs = dict(self.layout.server_opt_kwargs(self.cfg.server_opt_id, self.params),
                      **self.layout.dp_kwargs(self.cfg.dp_mode, self.clip, self.noise, SEED))
        self.m = _DpModule(base, kwargs, self.feds, self.layout.offsets["dp"])
        L = ledger()
        sz = self.sz
        roles = [TRAINER | COMM] * R if kw.get("solo") else [COMM] * kw["n_comm"] + [TRAINER] * (R - kw["n_comm"])
        n_tr = sum(1 for x in roles if x & TRAINER)
        st = base.state_init_bytes(R, kw["n_comm"], kw["aggregate_count"], roles, n_tr)
        for r, rep in enumerate(self.replicas):
            self.view(r, "state", [sz["RoundState"]], torch.uint8).copy_(torch.frombuffer(bytearray(st), dtype=torch.uint8))
            self.view(r, "dp", [sz["DpPage"]], torch.uint8).zero_()
            for name in ("server_m", "server_v")[: self.cfg.server_state_vectors]:
                self.view(r, name, [n_params], torch.float32).zero_()
            lc = rep.host_ledger.config()
            lc.dp_clip, lc.dp_noise, lc.dp_seed = self.clip, self.noise, SEED
            rep.host_ledger = L.Ledger(lc)
            rep.host_ledger.Bootstrap(roles)
            rep.state_bytes = self.view(r, "state", [sz["RoundState"]], torch.uint8)
            rep.ring_bytes = self.view(r, "ring", [self.layout.ring_slots * sz["BlockRecord"]], torch.uint8)
        torch.cuda.synchronize()

    def dp_page(self, r: int):
        """(norms [R], scales [R], sigma, epoch word) of rank r's DpPage."""
        sz = self.sz
        raw = self.view(r, "dp", [sz["DpPage"]], torch.uint8).cpu().numpy()
        f = lambda off, n: raw[off:off + 4 * n].view(np.float32)   # noqa: E731
        return (f(sz["dp_norm_off"], self.R), f(sz["dp_scale_off"], self.R), f(sz["dp_sigma_off"], 1)[0],
                int(raw[sz["dp_epoch_off"]:sz["dp_epoch_off"] + 4].view(np.uint32)[0]))

    def fill(self, name: str, value: np.ndarray):
        for r in range(self.R):
            self.view(r, name, [self.P], torch.float32).copy_(torch.from_numpy(value))


def scaled_uploads(rng, trainers, P, g: np.ndarray):
    """Finite updates around g at three scales (L2 norms ~ 0.06, 6.4, 640 for P = 4136): a clip of 1
    clips some of them and leaves the others alone."""
    return {t: torch.from_numpy((g + rng.standard_normal(P).astype(np.float32) * np.float32(10.0 ** (k % 3 * 2 - 3)))
                                .astype(np.float32)).cuda() for k, t in enumerate(trainers)}


def run_checked_rounds(h: DpHarness, rng, n_rounds: int, crafted_last: bool = True):
    """n_rounds rounds; after each: every replica's norms are the sequential fp64 norms within 1 fp32 ulp
    and identical across replicas, and every replica's model is the oracle's bit for bit.  The last
    round (crafted_last) uploads NaN, infinities and signed zeros.  Returns the final global model."""
    R, P = h.R, h.P
    g = h.view(0, "global", [P], torch.float32).cpu().numpy()
    m, v = np.zeros(P, np.float32), np.zeros(P, np.float32)
    for rnd in range(n_rounds):
        roles = h.roles()
        trainers = [r for r in range(R) if roles[r] & TRAINER]
        comm = [r for r in range(R) if roles[r] & COMM]
        if crafted_last and rnd == n_rounds - 1:
            ups = crafted_uploads(rng, trainers, P, g, rnd)
        else:
            ups = scaled_uploads(rng, trainers, P, g)
        n_samples = {t: 100 + 7 * t for t in trainers}
        correct = {c: rng.integers(0, N_VAL + 1, size=len(trainers)).tolist() for c in comm}
        e = h.round(ups, correct, n_samples)
        assert h.drain() == [[]] * R                     # every host ledger accepts every record
        blk = h.replicas[0].host_ledger.blocks()[-1]
        assert blk["epoch"] == e and blk["selected"], blk
        sel = blk["selected"]
        norms, scales, sigma, ep = h.dp_page(0)
        assert ep == e + 1
        for r in range(1, R):
            n_r, s_r, sg_r, _ = h.dp_page(r)
            assert same(n_r, norms).all() and same(s_r, scales).all() and same([sg_r], [sigma]).all()
        for t in trainers:
            u = ups[t].cpu().numpy()
            ref = dp_norm((u - g).astype(np.float32))
            if np.isfinite(ref):
                assert abs(float(norms[t]) - float(ref)) <= float(np.spacing(ref)), (rnd, t, norms[t], ref)
            else:
                assert same([norms[t]], [ref]).all(), (rnd, t, norms[t], ref)
        if rnd < n_rounds - 1 or not crafted_last:
            assert (scales[trainers] < 1).any() and (scales[trainers] == 1).any(), scales   # both kinds
        vals = np.stack([h.view(t, f"upload_master{e & 1}", [P], torch.float32).cpu().numpy() for t in sel])
        a = dp_device_combine(g, vals, blk["weight"], norms[sel], h.aggregation, h.trim, h.clip, h.noise, SEED, e)
        if h.server_opt != "none":
            g, m, v = server_step(g, a, m, v, h.server_opt, h.params)
        else:
            g = a
        g_b16 = torch.from_numpy(g).to(torch.bfloat16).float().numpy()
        for r in range(R):
            for reg, b16 in (("global", "global_shadow"), ("work_master", "work_shadow")):
                got = h.view(r, reg, [P], torch.float32).cpu().numpy()
                ok = same(got, g)
                assert ok.all(), (f"round {rnd} rank {r} {reg}: {int((~ok).sum())} coords differ, first "
                                  f"{np.flatnonzero(~ok)[:4]} got {got[~ok][:4]} want {g[~ok][:4]}")
                assert same(h.view(r, b16, [P], torch.bfloat16).float().cpu().numpy(), g_b16).all()
    return g


CASES = [  # (R, n_comm, aggregate_count, solo)
    (2, 2, 2, True),
    (4, 1, 3, False),
    (8, 2, 5, False),
]


def _params():
    out = []
    for R, nc, ag, solo in CASES:
        rules = [("fedavg", 1), ("median", 1)] + [("trimmed_mean", 1)] * (ag >= 3)
        for rule, trim in rules:
            for noise in ((0.0, 1.1) if rule == "fedavg" else (0.0,)):
                for opt in ("none", "adam"):
                    for ts in (False, True):
                        out.append(pytest.param(R, nc, ag, solo, rule, trim, noise, opt, ts,
                                                id=f"R{R}-{rule}-{'noise' if noise else 'clip'}-{opt}-"
                                                   f"{'two' if ts else 'one'}shot"))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("R,n_comm,agg,solo,rule,trim,noise,opt,two_shot", _params())
def test_harness_dp_round_matches_oracle(R, n_comm, agg, solo, rule, trim, noise, opt, two_shot):
    P = 8 * 517                                   # odd float4 count: uneven slices
    h = DpHarness(R, P, n_comm=n_comm, aggregate_count=agg, solo=solo, aggregation=rule, trim=trim,
                  two_shot=two_shot, server_opt=opt, clip=1.0, noise=noise)
    rng = np.random.default_rng(R * 1000 + len(rule) * 10 + int(noise * 10) + len(opt) + two_shot)
    g0 = (rng.standard_normal(P) * 0.5).astype(np.float32)
    for reg in ("global", "work_master", "upload_master0", "upload_master1"):
        h.fill(reg, g0)
    run_checked_rounds(h, rng, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("rule,noise", [("fedavg", 0.0), ("fedavg", 0.7), ("median", 0.0)])
def test_two_shot_equals_one_shot(rule, noise):
    P, R = 8 * 517, 4
    out = []
    for ts in (False, True):
        h = DpHarness(R, P, n_comm=1, aggregate_count=3, aggregation=rule, two_shot=ts, clip=1.0, noise=noise)
        rng = np.random.default_rng(21)
        g0 = (rng.standard_normal(P) * 0.5).astype(np.float32)
        for reg in ("global", "work_master", "upload_master0", "upload_master1"):
            h.fill(reg, g0)
        out.append(run_checked_rounds(h, rng, 3, crafted_last=False))
    assert same(out[0], out[1]).all()


@pytest.mark.gpu
def test_pure_noise_round_is_gaussian():
    """Every upload equal to g = 0: the FedAvg aggregate is exactly 0 and g' = sigma * xi.  g' / sigma passes
    a KS test against N(0, 1) over 2^20 coordinates; the next epoch (g reset to 0) draws other noise, with a
    correlation within 5 standard errors of 0."""
    from scipy import stats
    P, R = 1 << 20, 4
    h = DpHarness(R, P, n_comm=1, aggregate_count=3, clip=1.0, noise=1.0)
    zero = np.zeros(P, np.float32)
    draws = []
    for rnd in range(2):
        for reg in ("global", "work_master"):
            h.fill(reg, zero)
        trainers = [r for r in range(R) if h.roles()[r] & TRAINER]
        comm = [r for r in range(R) if h.roles()[r] & COMM]
        ups = {t: torch.zeros(P, device="cuda") for t in trainers}
        e = h.round(ups, {c: [N_VAL] * len(trainers) for c in comm}, {t: 100 for t in trainers})
        assert h.drain() == [[]] * R
        norms, scales, sigma, _ = h.dp_page(0)
        assert (norms[trainers] == 0).all() and (scales[trainers] == 1).all()
        assert sigma == np.float32(np.float32(1.0) * max(np.float32(w) for w in h.replicas[0].host_ledger.blocks()[-1]["weight"]))
        got = h.view(0, "global", [P], torch.float32).cpu().numpy()
        assert same(got, (sigma * dp_gauss(SEED, e, 0, P)).astype(np.float32)).all()
        z = got.astype(np.float64) / float(sigma)
        assert stats.kstest(z, "norm").pvalue > 1e-3, rnd
        draws.append(z)
    r = float(np.corrcoef(draws[0], draws[1])[0, 1])
    assert abs(r) < 5.0 / math.sqrt(P), r


@pytest.mark.gpu
def test_byzantine_update_is_bounded_by_the_clip():
    """R = 8, every trainer selected, one upload at 1e3 times an honest step: with the clip (noise 0) the
    model moves at most C * sum w_k plus the rounding of the fp32 combine, which is relative to |g| (each
    of the K fmaf steps and each clipped coordinate rounds once: (2K + 2) u (|g| + C)); without the clip
    it moves by hundreds."""
    P, R, C = 8 * 256, 8, 1.0
    moves = {}
    for clip in (C, None):
        h = (DpHarness(R, P, n_comm=2, aggregate_count=6, clip=clip) if clip else
             ServerOptHarness(R, P, n_comm=2, aggregate_count=6, server_opt="none"))
        rng = np.random.default_rng(5)
        g0 = (rng.standard_normal(P) * 0.5).astype(np.float32)
        for r in range(R):
            for reg in ("global", "work_master", "upload_master0", "upload_master1"):
                h.view(r, reg, [P], torch.float32).copy_(torch.from_numpy(g0))
        trainers = list(range(2, R))
        ups = {t: (g0 + rng.standard_normal(P).astype(np.float32) * np.float32(0.01)).astype(np.float32) for t in trainers}
        ups[7] = (g0 - np.float32(1e3) * (ups[7] - g0)).astype(np.float32)
        h.round({t: torch.from_numpy(u).cuda() for t, u in ups.items()}, {c: [N_VAL] * 6 for c in (0, 1)},
                {t: 100 for t in trainers})
        assert h.drain() == [[]] * R
        blk = h.replicas[0].host_ledger.blocks()[-1]
        assert 7 in blk["selected"] and len(blk["selected"]) == 6
        got = h.view(3, "global", [P], torch.float32).cpu().numpy()
        moves[clip] = float(np.linalg.norm(got.astype(np.float64) - g0))
        if clip:
            u, K = 2.0 ** -24, len(blk["selected"])
            bound = C * sum(blk["weight"]) * (1 + 8 * u) + (2 * K + 2) * u * (float(np.linalg.norm(g0)) + C)
            assert moves[clip] <= bound, (moves[clip], bound)
    assert moves[None] > 100 * moves[C], moves


# ------------------------------------------------------------------ engines, solo mode
def _check_engine_rounds(eng, run, n_rounds: int):
    """Genesis -> capture() (a real round) -> n_rounds - 1 more: after each, the model is the oracle's DP
    combine of the round's only upload (weight 1) from the previous model, with the device's norm."""
    P, cfg = eng.n_params, eng.cfg
    g = eng.global_master.cpu().numpy()
    clip, noise = (float(x) for x in cfg.dp_constants)
    for i in range(n_rounds):
        if i == 0:
            eng.capture()
        else:
            run()
        torch.cuda.synchronize()
        assert eng.drain_blocks() == []
        e = eng.read_state()["epoch"] - 1
        up = eng.heap.view(eng.layout.offsets[f"upload_master{e & 1}"], [P], torch.float32).cpu().numpy()
        norms = eng.last_update_norms()
        assert norms.shape == (1,) and abs(float(norms[0]) - float(dp_norm(up - g))) <= float(np.spacing(norms[0]))
        g = dp_device_combine(g, up[None], [1.0], norms, "fedavg", 1, clip, noise, eng.dp_seed, e)
        assert same(eng.global_master.cpu().numpy(), g).all(), i
        assert same(eng.work_master.cpu().numpy(), g).all()
    assert eng.read_state()["epoch"] == n_rounds


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_fused_engine_solo_dp(dtype):
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine

    shard = femnist_like(1, 512, seed=3)[0]
    kw = dict(hidden=256, batch_size=128, samples_per_client=512, learning_rate=0.01, dtype=dtype)
    off = FusedEngine(FLConfig.for_world(1, **kw), shard, rank=0, world=1, device=0)
    off.capture()
    base = off.launches_per_round             # 6 at N = 1 for fp8 (the default config), 5 for bf16
    assert base == (6 if dtype == "fp8" else 5) and off.last_update_norms() is None
    del off
    cfg = FLConfig.for_world(1, dp_clip=0.05, dp_noise=0.5, dp_seed=SEED, **kw)
    eng = FusedEngine(cfg, shard, rank=0, world=1, device=0)
    _check_engine_rounds(eng, eng.run_round_e2e, 3)
    assert eng.launches_per_round == base + 1      # fed_update_norms
    eps, delta = eng.privacy_spent()
    assert delta == 1e-5 and 0 < eps < math.inf
    # clip only: no noise, no privacy claim; the seed is not even drawn
    eng2 = FusedEngine(FLConfig.for_world(1, dp_clip=0.05, **kw), shard, rank=0, world=1, device=0)
    _check_engine_rounds(eng2, eng2.run_round_e2e, 2)
    assert eng2.privacy_spent()[0] == math.inf and eng2.dp_seed == 0


def _generic(**kw):
    from bflc_demo_b200.data.synthetic import cifar_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import LeNet5

    cfg = FLConfig.for_world(1, model="lenet5", dataset="cifar10", batch_size=64, samples_per_client=128,
                             learning_rate=0.01, **kw)
    shard = cifar_like(1, 128, seed=3, alpha=0.0)[0]
    return GenericFedEngine(cfg, LeNet5(10), shard, rank=0, world=1, device=0)


@pytest.mark.gpu
def test_generic_engine_solo_dp():
    eng = _generic(dp_clip=0.05, dp_noise=0.5, dp_seed=SEED)
    _check_engine_rounds(eng, eng.run_round, 3)
    # dp_seed None: a secret seed, drawn at construction
    a, b = _generic(dp_clip=0.05, dp_noise=0.5), _generic(dp_clip=0.05, dp_noise=0.5)
    assert a.dp_seed != b.dp_seed and a.host_ledger.config().dp_seed == a.dp_seed


@pytest.mark.gpu
def test_checkpoint_resume_continues_the_noise(tmp_path):
    """2 rounds, checkpoint, restore into a fresh engine, 2 more rounds: each round after the restore is
    the oracle's DP combine from the saved model with the saved seed's noise of that epoch.  (Local
    training is not bit-reproducible from run to run -- fp32 atomics -- so the rounds are compared with
    the oracle, as in test_gpu_server_optimizer.py.)"""
    from bflc_demo_b200.utils.checkpoint import load_checkpoint, save_checkpoint

    a = _generic(dp_clip=0.05, dp_noise=0.5)                      # a secret seed
    for _ in range(2):
        a.run_round()
    save_checkpoint(str(tmp_path / "ck.pt"), a)
    b = _generic(dp_clip=0.05, dp_noise=0.5)                      # another secret seed: adopts the saved one
    assert b.dp_seed != a.dp_seed
    assert load_checkpoint(str(tmp_path / "ck.pt"), b)["epoch"] == 2
    assert b.dp_seed == a.dp_seed and b.host_ledger.config().dp_seed == a.dp_seed
    g = a.global_master.cpu().numpy()
    assert same(b.global_master.cpu().numpy(), g).all()
    P = b.n_params
    for _ in range(2):
        b.run_round()
        torch.cuda.synchronize()
        e = b.read_state()["epoch"] - 1
        up = b.heap.view(b.layout.offsets[f"upload_master{e & 1}"], [P], torch.float32).cpu().numpy()
        g = dp_device_combine(g, up[None], [1.0], b.last_update_norms(), "fedavg", 1, 0.05, 0.5, a.dp_seed, e)
        assert same(b.global_master.cpu().numpy(), g).all()
    assert b.drain_blocks() == [] and b.read_state()["epoch"] == 4 and b.host_ledger.verify_chain()
    # a checkpoint restores only into an engine with the same DP settings and seed
    for other in (_generic(dp_clip=0.05), _generic(dp_clip=0.1, dp_noise=0.5), _generic(dp_clip=0.05, dp_noise=0.6),
                  _generic(), _generic(dp_clip=0.05, dp_noise=0.5, dp_seed=a.dp_seed ^ 1)):
        with pytest.raises(ValueError, match="differential privacy"):
            load_checkpoint(str(tmp_path / "ck.pt"), other)


@pytest.mark.gpu
def test_multi_gpu_dp_check():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs 2 GPUs")
    n = min(n, 8)
    cmd = [sys.executable, "-m", "torch.distributed.run", f"--nproc_per_node={n}",
           str(ROOT / "scripts" / "multi_gpu_check.py"), "dp"]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1800,
                       env=dict(os.environ, PYTHONPATH=str(ROOT)))
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    line = [ln for ln in p.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    res = json.loads(line[len("RESULT "):])["dp"]
    for name, r in res.items():
        assert r["errs"] == [] and r["identical"] and r["bit_exact"] and r["norms_ok"] and r["bounded"], (name, r)
