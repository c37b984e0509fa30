"""Adaptive clipping on the GPU: the adaptive k_consensus_dp kernels through the one-GPU replica harness of
test_gpu_dp.py, quantile tracking on the device, the engines in solo mode and a checkpoint / resume.

Every round is recomputed with the numpy oracle from the previous global model, the selected uploads, the
device's own norms and the oracle's own clip trajectory (``dp_clip_round``), and compared bit for bit: the
clip record (C_t, b~, n_sel) of every replica, its next clip, and its model."""
from __future__ import annotations

import functools
import math
import sys
from pathlib import Path
from unittest import mock

import numpy as np
import pytest
import torch

from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.protocol.oracle import dp_clip_round, dp_device_combine, dp_gauss, dp_norm, server_step

sys.path.insert(0, str(Path(__file__).resolve().parent))
from test_gpu_dp import SEED, DpHarness, scaled_uploads  # noqa: E402
from test_gpu_robust_aggregation import COMM, N_VAL, TRAINER, same  # noqa: E402

F = np.float32


class DpAdaptiveHarness(DpHarness):
    """DpHarness with adaptive clipping: its heaps are laid out with the DpAdapt header and the clip-record
    ring after the DpPage, genesis writes C_0 into every replica, and the host ledgers re-execute the clip
    trajectory from the drained records."""

    def __init__(self, R: int, n_params: int, *, clip: float, noise: float = 0.0, quantile: float = 0.5,
                 clip_lr: float = 0.2, count_noise: float = 0.0, **kw):
        from bflc_demo_b200._native import ledger
        from bflc_demo_b200.parallel import layout

        # the same harness, every dp layout it builds with the adaptive regions
        with mock.patch.object(layout, "HeapLayout", functools.partial(layout.HeapLayout, dp_adaptive=True)):
            super().__init__(R, n_params, clip=clip, noise=noise, **kw)
        lay = self.layout
        assert lay.dp_adaptive
        self.cfg = FLConfig(server_opt=self.server_opt, dp_clip=clip, dp_noise=noise, dp_seed=SEED,
                            dp_clip_quantile=quantile, dp_clip_lr=clip_lr, dp_count_noise=count_noise,
                            aggregation=self.aggregation, aggregate_count=kw["aggregate_count"],
                            needed_updates=kw["aggregate_count"], trim=self.trim).validate()
        self.q, self.lr, self.sb = (float(x) for x in self.cfg.dp_adapt_constants)
        self.m._kw.update(lay.dp_kwargs(self.cfg.dp_mode, self.clip, self.noise, SEED, adaptive=True))
        head, ring = lay.dp_adapt_offsets()
        hdr = self.m.dp_adapt_bytes(self.clip, self.noise, self.q, self.lr, self.sb)
        L = ledger()
        for r, rep in enumerate(self.replicas):
            self._raw(r, head, len(hdr)).copy_(torch.frombuffer(bytearray(hdr), dtype=torch.uint8))
            self._raw(r, ring, lay.ring_slots * self.sz["DpClipRecord"]).zero_()
            lc = rep.host_ledger.config()
            lc.dp_clip_quantile, lc.dp_clip_lr, lc.dp_count_noise = self.q, self.lr, self.sb
            roles = rep.host_ledger.roles()
            rep.host_ledger = L.Ledger(lc)
            rep.host_ledger.Bootstrap(roles)
        torch.cuda.synchronize()

    def _raw(self, r: int, off: int, n: int) -> torch.Tensor:
        return self.m.tensor_from_ptr(self.ptrs[r] + off, [n], torch.uint8, 0)

    def clip_now(self, r: int) -> np.float32:
        head, _ = self.layout.dp_adapt_offsets()
        return self._raw(r, head, 4).cpu().numpy().view(F)[0]

    def clip_record(self, r: int, e: int):
        """(seq, C_t, b~, n_sel) of epoch e on replica r."""
        from bflc_demo_b200.engine.base import CLIP_RECORD
        _, ring = self.layout.dp_adapt_offsets()
        raw = self._raw(r, ring, self.layout.ring_slots * CLIP_RECORD.size).cpu().numpy()
        return CLIP_RECORD.unpack_from(raw, (e % self.layout.ring_slots) * CLIP_RECORD.size)

    def drain(self):
        from bflc_demo_b200.engine.base import drain_ring
        torch.cuda.synchronize()
        _, ring = self.layout.dp_adapt_offsets()
        n = self.layout.ring_slots * self.sz["DpClipRecord"]
        errs = []
        for r, rep in enumerate(self.replicas):
            rep.drained, e = drain_ring(rep.host_ledger, rep.ring_bytes.cpu().numpy(), rep.drained,
                                        self.read_state(r)["epoch"], self.R, self._raw(r, ring, n).cpu().numpy())
            errs.append(e)
        return errs


def run_adaptive_rounds(h: DpAdaptiveHarness, rng, n_rounds: int, uploads=scaled_uploads):
    """n_rounds rounds checked against the oracle; returns the clip trajectory [C_0 .. C_n]."""
    R, P = h.R, h.P
    g = h.view(0, "global", [P], torch.float32).cpu().numpy()
    m, v = np.zeros(P, F), np.zeros(P, F)
    clip = F(h.clip)
    traj = [clip]
    for rnd in range(n_rounds):
        roles = h.roles()
        trainers = [r for r in range(R) if roles[r] & TRAINER]
        comm = [r for r in range(R) if roles[r] & COMM]
        ups = uploads(rng, trainers, P, g)
        correct = {c: rng.integers(0, N_VAL + 1, size=len(trainers)).tolist() for c in comm}
        e = h.round(ups, correct, {t: 100 + 7 * t for t in trainers})
        assert h.drain() == [[]] * R                      # every ledger re-executes the clip step
        blk = h.replicas[0].host_ledger.blocks()[-1]
        sel = blk["selected"]
        norms, _, _, _ = h.dp_page(0)
        for t in trainers:
            ref = dp_norm((ups[t].cpu().numpy() - g).astype(F))
            assert abs(float(norms[t]) - float(ref)) <= float(np.spacing(ref)), (rnd, t)
        count, nxt = dp_clip_round(norms[sel], clip, h.q, h.lr, h.sb, SEED, e)
        for r in range(R):
            seq, c_r, b_r, n_r = h.clip_record(r, e)
            assert (seq, n_r) == (e + 1, len(sel)) and same(c_r, clip) and same(b_r, count), (rnd, r)
            assert same(h.clip_now(r), nxt) and same(h.replicas[r].host_ledger.dp_clip_now(), nxt)
        vals = np.stack([h.view(t, f"upload_master{e & 1}", [P], torch.float32).cpu().numpy() for t in sel])
        a = dp_device_combine(g, vals, blk["weight"], norms[sel], h.aggregation, h.trim, clip, h.noise, SEED, e,
                              count_noise=h.sb)
        g, m, v = server_step(g, a, m, v, h.server_opt, h.params) if h.server_opt != "none" else (a, m, v)
        for r in range(R):
            for reg in ("global", "work_master"):
                assert same(h.view(r, reg, [P], torch.float32).cpu().numpy(), g).all(), (rnd, r, reg)
        clip = nxt
        traj.append(clip)
    return traj


CASES = [(2, 2, 2, True), (4, 1, 3, False)]


def _params():
    out = []
    for R, nc, ag, solo in CASES:
        rules = [("fedavg", 1), ("median", 1)] + [("trimmed_mean", 1)] * (ag >= 3)
        for rule, trim in rules:
            for noise in ((0.0, 1.1) if rule == "fedavg" else (0.0,)):
                for opt in (("none", "adam") if rule == "fedavg" else ("none",)):
                    for ts in (False, True):
                        out.append(pytest.param(R, nc, ag, solo, rule, trim, noise, opt, ts,
                                                id=f"R{R}-{rule}-{'noise' if noise else 'clip'}-{opt}-"
                                                   f"{'two' if ts else 'one'}shot"))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("R,n_comm,agg,solo,rule,trim,noise,opt,two_shot", _params())
def test_harness_adaptive_round_matches_oracle(R, n_comm, agg, solo, rule, trim, noise, opt, two_shot):
    P = 8 * 517
    h = DpAdaptiveHarness(R, P, n_comm=n_comm, aggregate_count=agg, solo=solo, aggregation=rule, trim=trim,
                          two_shot=two_shot, server_opt=opt, clip=1.0, noise=noise, quantile=0.3, clip_lr=0.5,
                          count_noise=2.0 if noise else 0.0)
    rng = np.random.default_rng(R * 100 + len(rule) + int(noise * 10) + len(opt) + two_shot)
    g0 = (rng.standard_normal(P) * 0.5).astype(F)
    for reg in ("global", "work_master", "upload_master0", "upload_master1"):
        h.fill(reg, g0)
    traj = run_adaptive_rounds(h, rng, 12)
    # a 0.3-quantile is never an equilibrium of 2 or 3 selected updates (b / n_sel in {0, 1/3, 1/2, 2/3, 1})
    assert len(set(float(c) for c in traj)) > 4


@pytest.mark.gpu
def test_count_noise_matches_the_host_sampler():
    """All-zero model changes: every norm is 0, b = n_sel, and b~ - n_sel is sigma_b times the host sampler's
    xi of (seed, epoch, kDpClipSite), bit for bit, on every replica."""
    P, R = 8 * 64, 4
    h = DpAdaptiveHarness(R, P, n_comm=1, aggregate_count=3, clip=1.0, noise=1.0, count_noise=3.0)
    zero = np.zeros(P, F)
    for rnd in range(3):
        for reg in ("global", "work_master"):
            h.fill(reg, zero)
        trainers = [r for r in range(R) if h.roles()[r] & TRAINER]
        comm = [r for r in range(R) if h.roles()[r] & COMM]
        e = h.round({t: torch.zeros(P, device="cuda") for t in trainers}, {c: [N_VAL] * 3 for c in comm},
                    {t: 100 for t in trainers})
        assert h.drain() == [[]] * R
        xi = dp_gauss(SEED, e, 0, 1, 0xDC000000)[0]
        for r in range(R):
            _, _, b, n = h.clip_record(r, e)
            assert n == 3 and same(b, F(F(3) + F(F(3.0) * xi)))


@pytest.mark.gpu
@pytest.mark.parametrize("start", [1e-2, 1e5])
def test_clip_tracks_the_quantile_on_the_device(start):
    """R = 8, six selected updates at the three scaled_uploads scales (norms ~ 0.064, 6.4, 640, two each):
    from 100x below and far above, C moves into the band between the small and the large norms, and its
    geometric mean over the last 10 rounds is within a factor 3 of the middle norms (the 0.5-quantile)."""
    P, R = 8 * 517, 8
    h = DpAdaptiveHarness(R, P, n_comm=2, aggregate_count=6, clip=start, quantile=0.5, clip_lr=1.0)
    rng = np.random.default_rng(11)
    g0 = (rng.standard_normal(P) * 0.5).astype(F)
    for reg in ("global", "work_master", "upload_master0", "upload_master1"):
        h.fill(reg, g0)
    traj = run_adaptive_rounds(h, rng, 40)
    mid = 6.4
    assert 0.064 < traj[-1] < 640, traj
    gm = math.exp(np.mean(np.log(np.asarray(traj[-10:], np.float64))))
    assert mid / 3 < gm < mid * 3, (gm, traj[-12:])


# ------------------------------------------------------------------ engines, solo mode
def _check_engine_rounds(eng, run, n_rounds: int, capture: bool):
    """Rounds after which the model is the oracle's DP combine of the only upload (weight 1) at the oracle's
    clip, and the engine reports that clip and noised count; the ledger accepts every record."""
    P, cfg = eng.n_params, eng.cfg
    g = eng.global_master.cpu().numpy()
    _, noise = (float(x) for x in cfg.dp_constants)
    q, lr, sb = (float(x) for x in cfg.dp_adapt_constants)
    clip = F(eng.clip_now())
    for i in range(n_rounds):
        if capture and i == 0:
            eng.capture()
        else:
            run()
        torch.cuda.synchronize()
        assert eng.drain_blocks() == []
        e = eng.read_state()["epoch"] - 1
        up = eng.heap.view(eng.layout.offsets[f"upload_master{e & 1}"], [P], torch.float32).cpu().numpy()
        norms, c_dev, b_dev = eng.last_update_norms(with_clip=True)
        count, nxt = dp_clip_round(norms[:1], clip, q, lr, sb, eng.dp_seed, e)
        assert same(c_dev, clip) and same(b_dev, count) and same(eng.clip_now(), nxt), (i, c_dev, clip)
        assert same(eng.host_ledger.dp_clip_now(), nxt)
        g = dp_device_combine(g, up[None], [1.0], norms, "fedavg", 1, clip, noise, eng.dp_seed, e, count_noise=sb)
        assert same(eng.global_master.cpu().numpy(), g).all(), i
        clip = nxt
    return clip


@pytest.mark.gpu
@pytest.mark.parametrize("noise", [0.0, 0.5])
def test_fused_engine_solo_adaptive(noise):
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine

    shard = femnist_like(1, 512, seed=3)[0]
    kw = dict(hidden=256, batch_size=128, samples_per_client=512, learning_rate=0.01, dtype="bf16")
    cfg = FLConfig.for_world(1, dp_clip=0.05, dp_noise=noise, dp_seed=SEED, dp_clip_quantile=0.5,
                             dp_count_noise=0.5 if noise else 0.0, **kw)
    eng = FusedEngine(cfg, shard, rank=0, world=1, device=0)
    _check_engine_rounds(eng, eng.run_round_e2e, 5, capture=True)          # graph replay after the eager round
    if noise:                                                              # epsilon of DP-FedAvg at the total z
        from bflc_demo_b200.protocol.privacy import epsilon
        assert eng.privacy_spent() == (epsilon(float(F(noise)), 5, 1e-5), 1e-5)


def _generic(**kw):
    from bflc_demo_b200.data.synthetic import cifar_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import LeNet5

    cfg = FLConfig.for_world(1, model="lenet5", dataset="cifar10", batch_size=64, samples_per_client=128,
                             learning_rate=0.01, **kw)
    shard = cifar_like(1, 128, seed=3, alpha=0.0)[0]
    return GenericFedEngine(cfg, LeNet5(10), shard, rank=0, world=1, device=0)


ADAPT = dict(dp_clip=0.05, dp_noise=0.5, dp_clip_quantile=0.5, dp_clip_lr=0.5, dp_count_noise=0.5)


@pytest.mark.gpu
def test_generic_engine_solo_adaptive_and_epsilon():
    eng = _generic(dp_seed=SEED, **ADAPT)
    _check_engine_rounds(eng, eng.run_round, 4, capture=False)
    fixed = _generic(dp_seed=SEED, dp_clip=0.05, dp_noise=0.5)
    for _ in range(4):
        fixed.run_round()
    assert eng.privacy_spent() == fixed.privacy_spent()                    # the same epsilon at the same z


@pytest.mark.gpu
def test_checkpoint_resume_continues_the_clip_trajectory(tmp_path):
    from bflc_demo_b200.utils.checkpoint import load_checkpoint, save_checkpoint

    a = _generic(**ADAPT)
    for _ in range(3):
        a.run_round()
    save_checkpoint(str(tmp_path / "ck.pt"), a)
    saved_clip = a.clip_now()
    assert saved_clip != float(F(0.05))
    b = _generic(**ADAPT)
    b.run_round()                                                          # a warm-up round moves b's clip
    assert load_checkpoint(str(tmp_path / "ck.pt"), b)["epoch"] == 3
    assert b.clip_now() == saved_clip and b.host_ledger.dp_clip_now() == saved_clip and b.dp_seed == a.dp_seed
    _check_engine_rounds(b, b.run_round, 3, capture=False)
    assert b.drain_blocks() == [] and b.read_state()["epoch"] == 6 and b.host_ledger.verify_chain()
    for other in (dict(ADAPT, dp_clip_quantile=0.6), dict(ADAPT, dp_clip_lr=0.3), dict(ADAPT, dp_count_noise=0.6),
                  dict(dp_clip=0.05, dp_noise=0.5)):
        with pytest.raises(ValueError, match="differential privacy"):
            load_checkpoint(str(tmp_path / "ck.pt"), _generic(**other))


# ------------------------------------------------------------------ edge rounds on the device
def _exact_uploads(rng, trainers, P, g):
    """From g = 0: the first trainer's change is 0.5 e_0 (norm exactly 0.5), the second's ~ 0.064, the rest ~ 640."""
    out = {}
    for k, t in enumerate(trainers):
        u = g.copy()
        if k == 0:
            u[0] = u[0] + F(0.5)
        else:
            u = u + rng.standard_normal(P).astype(F) * F(1e-3 if k == 1 else 10.0)
        out[t] = torch.from_numpy(u.astype(F)).cuda()
    return out


def _zero_harness(**kw):
    P = 8 * 517
    h = DpAdaptiveHarness(4, P, n_comm=1, aggregate_count=3, clip=0.5, quantile=0.5, **kw)
    for reg in ("global", "work_master", "upload_master0", "upload_master1"):
        h.fill(reg, np.zeros(P, F))
    return h


@pytest.mark.gpu
@pytest.mark.parametrize("noise", [0.0, 1.1])
def test_a_norm_equal_to_the_clip_is_counted(noise):
    """One update's device norm is exactly C = 0.5: it is not clipped and it is counted (b = 2 of 3)."""
    sb = 2.0 if noise else 0.0
    h = _zero_harness(noise=noise, count_noise=sb)
    trainers = [r for r in range(h.R) if h.roles()[r] & TRAINER]
    run_adaptive_rounds(h, np.random.default_rng(4), 1, uploads=_exact_uploads)
    norms, scales, _, _ = h.dp_page(0)
    assert norms[trainers[0]] == F(0.5) and scales[trainers[0]] == F(1.0)
    for r in range(h.R):
        seq, clip, count, n_sel = h.clip_record(r, 0)
        assert (seq, clip, n_sel) == (1, 0.5, 3)
        want = F(2) if sb == 0 else F(F(2) + F(F(sb) * dp_gauss(SEED, 0, 0, 1, 0xDC000000)[0]))
        assert same(count, want), (r, count, want)


def _set_n_aggregate(h, k: int):
    """Overwrite every replica's RoundState n_aggregate (word 3) with k."""
    for r in range(h.R):
        st = h.view(r, "state", [h.sz["RoundState"]], torch.uint8)
        st[12:16].view(torch.int32).fill_(k)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_fewer_selected_than_aggregate_count():
    """The device's n_aggregate is 8 with 3 trainers: every round selects n_sel = 3 < 8, and the clip step divides
    the noised count by n_sel (the oracle and every host ledger agree bit for bit over 6 rounds)."""
    h = _zero_harness(noise=1.1, count_noise=2.0)
    _set_n_aggregate(h, 8)
    traj = run_adaptive_rounds(h, np.random.default_rng(8), 6)
    for e in range(6):
        assert h.clip_record(0, e)[3] == 3
    assert len(set(float(c) for c in traj)) > 2


@pytest.mark.gpu
@pytest.mark.parametrize("noise", [0.0, 1.1])
def test_empty_round_keeps_the_clip(noise):
    """n_aggregate 0 on the device: the round selects nothing, so the model, C and the record's count stay put and
    nothing is drawn.  (No ledger configuration selects nothing, so the host ledger is not asked to re-execute it.)"""
    h = _zero_harness(noise=noise, count_noise=2.0 if noise else 0.0)
    rng = np.random.default_rng(6)
    run_adaptive_rounds(h, rng, 1, uploads=_exact_uploads)    # a normal round first: C moves away from C_0
    c1 = h.clip_now(0)
    g1 = h.view(0, "global", [h.P], torch.float32).cpu().numpy()
    _set_n_aggregate(h, 0)
    trainers = [r for r in range(h.R) if h.roles()[r] & TRAINER]
    comm = [r for r in range(h.R) if h.roles()[r] & COMM]
    e = h.round(scaled_uploads(rng, trainers, h.P, g1), {c: [N_VAL] * 3 for c in comm}, {t: 100 for t in trainers})
    for r in range(h.R):
        assert h.clip_record(r, e) == (e + 1, float(c1), 0.0, 0) and same(h.clip_now(r), c1)
        assert same(h.view(r, "global", [h.P], torch.float32).cpu().numpy(), g1).all()


@pytest.mark.gpu
def test_adaptive_mode_needs_the_adaptive_layout():
    """Kernel modes 3 / 4 write past the DpPage: the binding refuses a dp region without those regions."""
    h = DpHarness(2, 8 * 64, n_comm=2, aggregate_count=2, solo=True, clip=1.0)
    for mode in (1, 2):
        kw = h.layout.dp_kwargs(mode, 1.0, 1.0 if mode == 2 else 0.0, SEED, adaptive=True)
        with pytest.raises(RuntimeError, match="adaptive clipping"):
            h.m._mod.fed_consensus_aggregate(h.feds[0], N_VAL, False, False, False, **kw)
