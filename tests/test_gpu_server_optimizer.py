"""Server optimizers (FedAvgM momentum, FedAdam, FedYogi) on the GPU: the consensus kernel's step on
the aggregate, checked through the one-GPU replica harness of test_gpu_robust_aggregation.py, the
engines in solo mode, a checkpoint / resume, and (4+ GPUs) the multi-GPU check.

Every check recomputes the step with the numpy oracle (protocol/oracle.py ``server_step``) from the
previous global model and the round's aggregate, both read back from the heaps, and compares bit for
bit (NaN compared as NaN)."""
from __future__ import annotations

import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.protocol.oracle import aggregation_trim, robust_combine, server_step

sys.path.insert(0, str(Path(__file__).resolve().parent))
from test_gpu_robust_aggregation import (COMM, N_VAL, TRAINER, ReplicaHarness, crafted_uploads,  # noqa: E402
                                         fedavg_reference, same)

ROOT = Path(__file__).resolve().parents[1]
OPTS = ["momentum", "adam", "yogi"]


def two_shot_slice(P: int, R: int, r: int):
    """Elements [lo, hi) rank r reduces in two-shot mode (k_consensus: even float4 slices)."""
    nv = P // 4
    per = (nv + R - 1) // R
    per += per & 1
    lo = min(per * r, nv)
    return 4 * lo, 4 * min(lo + per, nv)


class _ServerOptModule:
    """The native module, with the server optimizer's arguments added to every consensus launch (the
    state offsets are relative to each rank's own heap, so they are the same for every rank)."""

    def __init__(self, mod, kw: dict):
        self._mod, self._kw = mod, kw

    def __getattr__(self, name):
        return getattr(self._mod, name)

    def fed_consensus_aggregate(self, *a, **kw):
        return self._mod.fed_consensus_aggregate(*a, **kw, **self._kw)


class ServerOptHarness(ReplicaHarness):
    """ReplicaHarness whose heaps carry server optimizer state and whose host ledgers expect the
    optimizer in every block record."""

    def __init__(self, R: int, n_params: int, *, server_opt: str, server_lr: float = 0.0, **kw):
        from bflc_demo_b200._native import ledger
        from bflc_demo_b200.parallel.layout import HeapLayout

        super().__init__(R, n_params, **kw)
        self.cfg = FLConfig(server_opt=server_opt, server_lr=server_lr).validate()
        self.server_opt, self.params = server_opt, self.cfg.server_opt_constants
        # the same harness over heaps laid out with the state regions (appended after every other
        # region, so every other offset is unchanged)
        self.layout = HeapLayout(n_params, self.layout.ring_slots, server_state=self.cfg.server_state_vectors)
        self.heaps = self.ptrs = None               # free the first heaps before allocating these
        self.heaps = [self.m.SymmHeap(self.layout.total_bytes, 0, 1, 0, "local") for _ in range(R)]
        self.ptrs = [h.local_ptr() for h in self.heaps]
        self.feds = [self.layout.fed_dict(r, R, self.ptrs, 0) for r in range(R)]
        self.m = _ServerOptModule(self.m, self.layout.server_opt_kwargs(self.cfg.server_opt_id, self.params))
        L = ledger()
        sz = self.sz
        roles = [TRAINER | COMM] * R if kw.get("solo") else [COMM] * kw["n_comm"] + [TRAINER] * (R - kw["n_comm"])
        n_tr = sum(1 for x in roles if x & TRAINER)
        st = self.m.state_init_bytes(R, kw["n_comm"], kw["aggregate_count"], roles, n_tr)
        want = self.cfg.to_ledger_config(n_params)
        for r, rep in enumerate(self.replicas):
            self.view(r, "state", [sz["RoundState"]], torch.uint8).copy_(torch.frombuffer(bytearray(st), dtype=torch.uint8))
            for name in ("server_m", "server_v")[: self.cfg.server_state_vectors]:
                self.view(r, name, [n_params], torch.float32).zero_()
            lc = rep.host_ledger.config()
            lc.server_opt, lc.server_lr, lc.server_beta1 = want.server_opt, want.server_lr, want.server_beta1
            lc.server_beta2, lc.server_tau = want.server_beta2, want.server_tau
            rep.host_ledger = L.Ledger(lc)
            rep.host_ledger.Bootstrap(roles)
            rep.state_bytes = self.view(r, "state", [sz["RoundState"]], torch.uint8)
            rep.ring_bytes = self.view(r, "ring", [self.layout.ring_slots * sz["BlockRecord"]], torch.uint8)
        torch.cuda.synchronize()

    def state(self, r: int):
        P = self.P
        m = self.view(r, "server_m", [P], torch.float32).cpu().numpy()
        v = (self.view(r, "server_v", [P], torch.float32).cpu().numpy() if self.server_opt != "momentum"
             else np.zeros(P, np.float32))
        return m, v


CASES = [  # (R, n_comm, aggregate_count, solo)
    (2, 2, 2, True),
    (4, 1, 3, False),
    (8, 2, 5, False),
]
PARAMS = [pytest.param(R, nc, ag, solo, opt, rule, ts, id=f"R{R}-{opt}-{rule}-{'two' if ts else 'one'}shot")
          for (R, nc, ag, solo) in CASES for opt in OPTS for rule in ("fedavg", "median") for ts in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("R,n_comm,agg,solo,opt,rule,two_shot", PARAMS)
def test_harness_server_step_matches_oracle(R, n_comm, agg, solo, opt, rule, two_shot):
    P = 8 * 517                                   # odd float4 count: uneven two-shot slices
    h = ServerOptHarness(R, P, n_comm=n_comm, aggregate_count=agg, solo=solo, aggregation=rule,
                         two_shot=two_shot, server_opt=opt, server_lr=0.5 if opt == "momentum" else 0.0)
    rng = np.random.default_rng(R * 100 + OPTS.index(opt) * 10 + len(rule) + 7 * two_shot)
    g0 = (rng.standard_normal(P) * 0.5).astype(np.float32)
    for r in range(R):
        for reg in ("global", "work_master", "upload_master0", "upload_master1"):
            h.view(r, reg, [P], torch.float32).copy_(torch.from_numpy(g0))
    g, m, v = g0, np.zeros(P, np.float32), np.zeros(P, np.float32)
    for rnd in range(3):
        roles = h.roles()
        trainers = [r for r in range(R) if roles[r] & TRAINER]
        comm = [r for r in range(R) if roles[r] & COMM]
        ups = crafted_uploads(rng, trainers, P, g, rnd)
        n_samples = {t: 100 + 7 * t for t in trainers}
        correct = {c: rng.integers(0, N_VAL + 1, size=len(trainers)).tolist() for c in comm}
        e = h.round(ups, correct, n_samples)
        errs = h.drain()
        assert errs == [[]] * R, errs                   # every host ledger accepts every record
        blk = h.replicas[0].host_ledger.blocks()[-1]
        assert blk["epoch"] == e and blk["selected"], blk
        vals = np.stack([h.view(t, f"upload_master{e & 1}", [P], torch.float32).cpu().numpy() for t in blk["selected"]])
        a = fedavg_reference(vals, blk["weight"]) if rule == "fedavg" else robust_combine(vals, aggregation_trim(rule, 1))
        g, m, v = server_step(g, a, m, v, opt, h.params)
        g_b16 = torch.from_numpy(g).to(torch.bfloat16).float().numpy()
        for r in range(R):
            for reg, b16 in (("global", "global_shadow"), ("work_master", "work_shadow")):
                got = h.view(r, reg, [P], torch.float32).cpu().numpy()
                ok = same(got, g)
                assert ok.all(), (f"round {rnd} rank {r} {reg}: {int((~ok).sum())} coords differ, first "
                                  f"{np.flatnonzero(~ok)[:4]} got {got[~ok][:4]} want {g[~ok][:4]}")
                gb = h.view(r, b16, [P], torch.bfloat16).float().cpu().numpy()
                assert same(gb, g_b16).all(), f"round {rnd} rank {r} {b16}: not the RNE of the fp32 result"
            lo, hi = two_shot_slice(P, R, r) if two_shot else (0, P)
            assert hi > lo
            sm, sv = h.state(r)
            assert same(sm[lo:hi], m[lo:hi]).all(), f"round {rnd} rank {r}: server_m differs in [{lo}, {hi})"
            if opt != "momentum":
                assert same(sv[lo:hi], v[lo:hi]).all(), f"round {rnd} rank {r}: server_v differs in [{lo}, {hi})"
    assert np.isfinite(g).any() and (m != 0).any()


@pytest.mark.gpu
@pytest.mark.parametrize("two_shot", [False, True], ids=["oneshot", "twoshot"])
@pytest.mark.parametrize("opt", ["adam", "yogi"])
def test_harness_subnormal_state_arithmetic(opt, two_shot):
    """Coordinates where d*d is just above the smallest normal and the preset v sits at, just above,
    just below, or a subnormal step away from it: v - d*d is 0 or subnormal and c2*(d*d) is
    subnormal.  The device (built with --use_fast_math) must keep them exactly like the oracle --
    in particular yogi's sign(v - d*d) must be +-1, not 0, for a subnormal difference."""
    R, P = 4, 8 * 517
    h = ServerOptHarness(R, P, n_comm=1, aggregate_count=3, aggregation="median", two_shot=two_shot,
                         server_opt=opt)
    rng = np.random.default_rng(17 + two_shot)
    f = np.float32
    g0 = (rng.standard_normal(P) * 0.5).astype(f)
    g_s, d_s = f(2e-19), f(1.378e-19)
    a_s = f(g_s - d_s)
    d = f(g_s - a_s)
    dd = f(d * d)
    assert dd >= np.finfo(f).tiny
    steps = [0, 1, 3, -1, -2]                                     # v = dd + k ulps (ulp of dd: 2^-149)
    v_special = [np.nextafter(dd, f(np.inf) if k > 0 else f(-np.inf), dtype=f) if k else dd for k in steps]
    for i, k in enumerate(steps):
        for _ in range(abs(k) - 1):
            v_special[i] = np.nextafter(v_special[i], f(np.inf) if k > 0 else f(-np.inf), dtype=f)
    v_special += [f(2e-38), f(np.nan)]
    idx = np.arange(len(v_special)) * 531 % P                      # spread over the two-shot slices
    with np.errstate(all="ignore"):
        diff = (np.array(v_special[:-1], f) - dd).astype(f)
    assert (diff == 0).any() and ((diff != 0) & (np.abs(diff) < np.finfo(f).tiny)).sum() >= 4
    g0[idx] = g_s
    v0 = np.zeros(P, f)
    v0[idx] = v_special
    trainers = [1, 2, 3]
    ups = {}
    for t in trainers:
        u = (g0 + rng.standard_normal(P).astype(f) * 0.1).astype(f)
        u[idx] = a_s
        ups[t] = torch.from_numpy(u).cuda()
    for r in range(R):
        for reg in ("global", "work_master", "upload_master0", "upload_master1"):
            h.view(r, reg, [P], torch.float32).copy_(torch.from_numpy(g0))
        h.view(r, "server_v", [P], torch.float32).copy_(torch.from_numpy(v0))
    e = h.round(ups, {0: [N_VAL] * 3}, {t: 100 for t in trainers})
    assert h.drain() == [[]] * R
    blk = h.replicas[0].host_ledger.blocks()[-1]
    assert blk["epoch"] == e and blk["selected"] == trainers
    vals = np.stack([h.view(t, f"upload_master{e & 1}", [P], torch.float32).cpu().numpy() for t in trainers])
    a = robust_combine(vals, aggregation_trim("median", 1))
    assert (a[idx] == a_s).all()
    g, m, v = server_step(g0, a, np.zeros(P, f), v0, opt, h.params)
    if opt == "yogi":                                             # the sign moved v wherever v != d*d
        assert (v[idx[1:5]] != v0[idx[1:5]]).all() and v[idx[0]] == v0[idx[0]]
    for r in range(R):
        assert same(h.view(r, "global", [P], torch.float32).cpu().numpy(), g).all(), r
        lo, hi = two_shot_slice(P, R, r) if two_shot else (0, P)
        sm, sv = h.state(r)
        bad = np.flatnonzero(~same(sv[lo:hi], v[lo:hi])) + lo
        assert bad.size == 0, (r, bad[:4], sv[bad[:4]], v[bad[:4]])
        assert same(sm[lo:hi], m[lo:hi]).all(), r


# ------------------------------------------------------------------ engines, solo mode
def _check_engine_rounds(eng, run, n_rounds: int, opt: str):
    """Genesis -> capture() (a real round) -> n_rounds - 1 more: after each, global and training copies
    are the oracle step from the previous global model and the round's (only) upload, and so is the state."""
    P = eng.n_params
    cfg = eng.cfg
    g = eng.global_master.cpu().numpy()
    m, v = np.zeros(P, np.float32), np.zeros(P, np.float32)
    for i in range(n_rounds):
        if i == 0:
            eng.capture()
        else:
            run()
        torch.cuda.synchronize()
        assert eng.drain_blocks() == []
        e = eng.read_state()["epoch"] - 1
        up = eng.heap.view(eng.layout.offsets[f"upload_master{e & 1}"], [P], torch.float32).cpu().numpy()
        g, m, v = server_step(g, up, m, v, opt, cfg.server_opt_constants)
        got = eng.global_master.cpu().numpy()
        assert same(got, g).all(), (i, np.flatnonzero(~same(got, g))[:4])
        assert same(eng.work_master.cpu().numpy(), g).all()
        assert same(eng.server_state[0].cpu().numpy(), m).all()
        if opt != "momentum":
            assert same(eng.server_state[1].cpu().numpy(), v).all()
    assert eng.read_state()["epoch"] == n_rounds and not np.array_equal(g, up)


@pytest.mark.gpu
@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_fused_engine_solo_server_opt(dtype, opt):
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine

    cfg = FLConfig.for_world(1, hidden=256, batch_size=128, samples_per_client=512, learning_rate=0.01, dtype=dtype,
                             server_opt=opt)
    shard = femnist_like(1, 512, seed=3)[0]
    eng = FusedEngine(cfg, shard, rank=0, world=1, device=0)
    _check_engine_rounds(eng, eng.run_round_e2e, 3, opt)


def _generic(opt, **kw):
    from bflc_demo_b200.data.synthetic import cifar_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import LeNet5

    cfg = FLConfig.for_world(1, model="lenet5", dataset="cifar10", batch_size=64, samples_per_client=128,
                             learning_rate=0.01, server_opt=opt, **kw)
    shard = cifar_like(1, 128, seed=3, alpha=0.0)[0]
    return GenericFedEngine(cfg, LeNet5(10), shard, rank=0, world=1, device=0)


@pytest.mark.gpu
@pytest.mark.parametrize("opt", OPTS)
def test_generic_engine_solo_server_opt(opt):
    eng = _generic(opt)
    _check_engine_rounds(eng, eng.run_round, 3, opt)


@pytest.mark.gpu
def test_checkpoint_resume_keeps_the_server_state(tmp_path):
    """Generic engine, adam: 2 rounds, checkpoint, restore into a fresh engine, 2 more rounds.  The
    restored model and state are the saved ones bit for bit, and every round after the restore is the
    oracle step from them.  (The local training itself is not bit-reproducible from run to run: its
    bias gradients and split-K GEMMs accumulate with fp32 atomics, so two uninterrupted runs already
    differ in the last bits, and the resumed run is compared with the oracle instead.)"""
    from bflc_demo_b200.utils.checkpoint import load_checkpoint, save_checkpoint

    a = _generic("adam")
    for _ in range(2):
        a.run_round()
    save_checkpoint(str(tmp_path / "ck.pt"), a)
    saved = [t.clone() for t in [a.global_master] + a.server_state]
    assert all(bool((t != 0).any()) for t in saved)
    b = _generic("adam")
    assert load_checkpoint(str(tmp_path / "ck.pt"), b)["epoch"] == 2
    for x, y in zip([b.global_master] + b.server_state, saved):
        assert torch.equal(x, y)
    g, m, v = (t.cpu().numpy() for t in saved)
    P = b.n_params
    for _ in range(2):
        b.run_round()
        torch.cuda.synchronize()
        e = b.read_state()["epoch"] - 1
        up = b.heap.view(b.layout.offsets[f"upload_master{e & 1}"], [P], torch.float32).cpu().numpy()
        g, m, v = server_step(g, up, m, v, "adam", b.cfg.server_opt_constants)
        assert same(b.global_master.cpu().numpy(), g).all()
        assert same(b.server_state[0].cpu().numpy(), m).all() and same(b.server_state[1].cpu().numpy(), v).all()
    assert b.drain_blocks() == [] and b.read_state()["epoch"] == 4 and b.host_ledger.verify_chain()
    # a checkpoint restores only into an engine with the same server optimizer
    for other in (_generic("yogi"), _generic("adam", server_beta2=0.999), _generic("none")):
        with pytest.raises(ValueError, match="server optimizer"):
            load_checkpoint(str(tmp_path / "ck.pt"), other)
    # ... compared on the hyperparameters it uses: momentum has no beta2 / tau
    c = _generic("momentum")
    c.run_round()
    save_checkpoint(str(tmp_path / "mom.pt"), c)
    d = _generic("momentum", server_beta2=0.5, server_tau=1.0)
    assert load_checkpoint(str(tmp_path / "mom.pt"), d)["epoch"] == 1
    assert torch.equal(d.server_state[0], c.server_state[0])
    with pytest.raises(ValueError, match="server optimizer"):
        load_checkpoint(str(tmp_path / "mom.pt"), _generic("momentum", server_beta1=0.5))


@pytest.mark.gpu
def test_multi_gpu_server_opt_check():
    n = torch.cuda.device_count()
    if n < 4:
        pytest.skip("needs 4 GPUs")
    n = 8 if n >= 8 else 4
    cmd = [sys.executable, "-m", "torch.distributed.run", f"--nproc_per_node={n}",
           str(ROOT / "scripts" / "multi_gpu_check.py"), "serveropt"]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1800,
                       env=dict(os.environ, PYTHONPATH=str(ROOT)))
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    line = [ln for ln in p.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    res = json.loads(line[len("RESULT "):])["serveropt"]
    assert set(k.split("_")[0] for k in res) == set(OPTS)
    for name, r in res.items():
        assert r["errs"] == [] and r["identical"] and r["bit_exact"] and r["state_exact"], (name, r)
