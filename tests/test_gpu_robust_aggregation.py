"""Byzantine-robust aggregation on the GPU: the consensus kernel's coordinate-wise median / trimmed
mean, checked through a one-GPU replica harness, the engines in solo mode, and (4+ GPUs) the
multi-GPU check.

The harness drives the real protocol kernels (fed_plan_round, fed_upload, fed_consensus_aggregate)
for R emulated ranks whose symmetric heaps are R plain allocations on one device.  Every launch is
sequential on one stream, so every flag a kernel polls must already be released by an earlier
launch; the harness asserts that on the host before each launch (a harness bug fails in Python and
never spins on the GPU).  Where a kernel waits for a rank that has not run yet -- a committee
rank's score row, a two-shot slice -- the harness writes that word itself first: score rows are
exact (n_val is a power of two), slice digests are ignored in that mode.  Multicast cannot be
emulated on one device and stays with scripts/multi_gpu_check.py."""
from __future__ import annotations

import json
import os
import subprocess
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from bflc_demo_b200.protocol.oracle import AGGREGATIONS, aggregation_trim, robust_combine

ROOT = Path(__file__).resolve().parents[1]
TRAINER, COMM = 1, 2
FLAG_TRAINED, FLAG_SCORED, FLAG_DONE, FLAG_SLICE = 0, 8, 16, 24
N_VAL = 64                       # committee scores correct / 64: exact in fp32


class ReplicaHarness:
    """R emulated ranks on one GPU, each with its own heap, ledger page and host ledger."""

    def __init__(self, R: int, n_params: int, *, n_comm: int, aggregate_count: int, solo: bool = False,
                 aggregation: str = "fedavg", trim: int = 1, two_shot: bool = False, ring_slots: int = 16):
        from bflc_demo_b200._native import C, ledger
        from bflc_demo_b200.parallel.layout import HeapLayout

        self.m = m = C()
        self.R, self.P, self.two_shot = R, n_params, two_shot
        self.rule, self.trim = AGGREGATIONS.index(aggregation), trim
        self.aggregation = aggregation
        self.sz = sz = m.struct_sizes()
        self.K = sz["kMaxRanks"]
        self.layout = HeapLayout(n_params, ring_slots)
        self.heaps = [m.SymmHeap(self.layout.total_bytes, 0, 1, 0, "local") for _ in range(R)]
        self.ptrs = [h.local_ptr() for h in self.heaps]
        self.feds = [self.layout.fed_dict(r, R, self.ptrs, 0) for r in range(R)]
        roles = [TRAINER | COMM] * R if solo else [COMM] * n_comm + [TRAINER] * (R - n_comm)
        n_tr = sum(1 for x in roles if x & TRAINER)
        st = m.state_init_bytes(R, n_comm, aggregate_count, roles, n_tr)
        L = ledger()
        self.replicas = []
        for r in range(R):
            self.view(r, "state", [sz["RoundState"]], torch.uint8).copy_(
                torch.frombuffer(bytearray(st), dtype=torch.uint8))
            lc = L.LedgerConfig()
            lc.client_num, lc.comm_count, lc.aggregate_count = R, n_comm, aggregate_count
            lc.needed_update_count, lc.model_size, lc.solo = n_tr, n_params, int(solo)
            lc.aggregation, lc.trim = self.rule, trim
            led = L.Ledger(lc)
            led.Bootstrap(roles)
            self.replicas.append(SimpleNamespace(
                host_ledger=led, drained=0, state_bytes=self.view(r, "state", [sz["RoundState"]], torch.uint8),
                ring_bytes=self.view(r, "ring", [ring_slots * sz["BlockRecord"]], torch.uint8)))
        torch.cuda.synchronize()

    def view(self, r: int, region: str, shape, dtype) -> torch.Tensor:
        return self.m.tensor_from_ptr(self.ptrs[r] + self.layout.offsets[region], list(shape), dtype, 0)

    def flags(self, r: int) -> torch.Tensor:
        return self.view(r, "flags", [self.sz["FLAG_COUNT"]], torch.int32)

    def read_state(self, r: int = 0) -> dict:
        from bflc_demo_b200.engine.base import parse_round_state
        return parse_round_state(self.replicas[r].state_bytes.cpu().numpy(), self.R)

    def roles(self):
        return self.read_state()["roles"]

    def epoch(self) -> int:
        return self.read_state()["epoch"]

    def _expect(self, r: int, words, target: int, what: str):
        torch.cuda.synchronize()
        f = self.flags(r).cpu().numpy()
        low = [w for w in words if int(f[w]) < target]
        assert not low, f"{what} on rank {r}: flag words {low} below {target} (harness order bug)"

    def round(self, uploads: dict, correct: dict, n_samples: dict, byz=(), events=None):
        """One round: uploads[t] = fp32 [P] work_master of trainer t, correct[c] = int32 [n_cand]
        validation counts of committee rank c.  ``events`` = (start, stop) CUDA events recorded
        around rank 0's consensus launch.  Returns the epoch that was closed."""
        m, R, K = self.m, self.R, self.K
        e = self.epoch()
        roles = self.roles()
        par = e & 1
        trainers = [r for r in range(R) if roles[r] & TRAINER]
        comm = [r for r in range(R) if roles[r] & COMM]
        for r in range(R):
            if e >= 2:
                self._expect(r, [FLAG_DONE + q for q in range(R)], e - 1, "fed_plan_round")
            m.fed_plan_round(self.feds[r], [], 1, False)
        for t in trainers:
            self.view(t, "work_master", [self.P], torch.float32).copy_(uploads[t])
            m.fed_upload(self.feds[t], int(n_samples[t]), 1, 1 if t in byz else 0, 5.0)
        for c in comm:
            self.view(c, "plan", [self.sz["RoundPlan"]], torch.uint8)[
                self.sz["plan_correct_off"]:self.sz["plan_correct_off"] + 4 * K].view(torch.int32)[
                : len(correct[c])].copy_(torch.as_tensor(correct[c], dtype=torch.int32))
        for r in range(R):
            fl = self.flags(r)
            for c in comm:
                if c > r:   # committee rank c has not run yet: its score row and flag, exactly
                    row = self.view(r, "scores", [2 * K * K], torch.float32)[(par * K + c) * K:(par * K + c + 1) * K]
                    for z, t in enumerate(trainers):
                        row[t] = float(correct[c][z]) / N_VAL
                    fl[FLAG_SCORED + c] = e + 1
            if self.two_shot:
                for q in range(r + 1, R):
                    fl[FLAG_SLICE + q] = e + 1
            # (a committee rank releases its own score flag itself before it waits)
            self._expect(r, [FLAG_SCORED + c for c in comm if c != r] + [FLAG_TRAINED + t for t in trainers],
                         e + 1, "fed_consensus_aggregate")
            if self.two_shot:
                self._expect(r, [FLAG_SLICE + q for q in range(R) if q != r], e + 1, "two-shot publish")
            if events is not None and r == 0:
                events[0].record()
            m.fed_consensus_aggregate(self.feds[r], N_VAL, False, self.two_shot, False,
                                      rule=self.rule, trim=self.trim)
            if events is not None and r == 0:
                events[1].record()
        torch.cuda.synchronize()
        return e

    def drain(self):
        """Every replica's device ring into its host ledger (the engines' drain_blocks); the mismatches
        by replica."""
        from bflc_demo_b200.engine.base import drain_ring
        torch.cuda.synchronize()
        errs = []
        for r, rep in enumerate(self.replicas):
            rep.drained, e = drain_ring(rep.host_ledger, rep.ring_bytes.cpu().numpy(), rep.drained,
                                        self.read_state(r)["epoch"], self.R)
            errs.append(e)
        return errs


def fedavg_reference(vals: np.ndarray, weights) -> np.ndarray:
    """The kernel's FedAvg: acc = fmaf(w_k, v_k, acc) in ascending rank order (fp64 product and sum
    are exact enough that one rounding to fp32 is the fused multiply-add)."""
    acc = np.zeros(vals.shape[1], np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for w, v in zip(weights, vals):
            acc = (np.float64(np.float32(w)) * v.astype(np.float64) + acc.astype(np.float64)).astype(np.float32)
    return acc


def same(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Bit equality, NaN compared as NaN."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def crafted_uploads(rng, trainers, P, global_now: np.ndarray, round_idx: int):
    """Random honest updates around the global model, plus NaN, +-inf, +-0 and exact ties."""
    base = np.nan_to_num(global_now, nan=0.0, posinf=0.0, neginf=0.0)
    ups = {t: (base + rng.standard_normal(P).astype(np.float32) * 0.1).astype(np.float32) for t in trainers}
    t0, t1 = trainers[0], trainers[-1]
    idx = rng.choice(P, size=48, replace=False)
    ups[t0][idx[:6]] = np.nan
    ups[t0][idx[6:12]] = np.inf
    ups[t1][idx[12:18]] = -np.inf
    ups[t0][idx[18:24]] = 0.0
    ups[t1][idx[24:30]] = -0.0
    for t in trainers:                               # ties: every trainer holds the same value
        ups[t][idx[30:36]] = np.float32(0.25 * (round_idx + 1))
    if len(trainers) > 1:                            # pairwise ties
        ups[trainers[1]][idx[36:48]] = ups[t0][idx[36:48]]
    return {t: torch.from_numpy(u).cuda() for t, u in ups.items()}


CASES = [  # (R, n_comm, aggregate_count, solo)
    (2, 2, 2, True),
    (4, 1, 3, False),
    (8, 2, 5, False),
]


def _rules(agg_count):
    """FedAvg, median, and every trim the ledger accepts (2 * trim < aggregate_count), up to 2."""
    return [("fedavg", 1), ("median", 1)] + [("trimmed_mean", t) for t in (1, 2) if 2 * t < agg_count]


PARAMS = [pytest.param(R, nc, ag, solo, rule, trim, ts, id=f"R{R}-{rule}{trim if rule == 'trimmed_mean' else ''}-"
                       f"{'two' if ts else 'one'}shot")
          for (R, nc, ag, solo) in CASES for (rule, trim) in _rules(ag) for ts in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("R,n_comm,agg,solo,rule,trim,two_shot", PARAMS)
def test_harness_rule_matches_reference(R, n_comm, agg, solo, rule, trim, two_shot):
    P = 8 * 517                                   # odd float4 count: uneven two-shot slices
    h = ReplicaHarness(R, P, n_comm=n_comm, aggregate_count=agg, solo=solo, aggregation=rule, trim=trim,
                       two_shot=two_shot)
    rng = np.random.default_rng(R * 100 + len(rule) + trim + 7 * two_shot)
    g0 = (rng.standard_normal(P) * 0.5).astype(np.float32)
    for r in range(R):
        for reg in ("global", "work_master", "upload_master0", "upload_master1"):
            h.view(r, reg, [P], torch.float32).copy_(torch.from_numpy(g0))
    for rnd in range(3):
        roles = h.roles()
        trainers = [r for r in range(R) if roles[r] & TRAINER]
        comm = [r for r in range(R) if roles[r] & COMM]
        global_now = h.view(0, "global", [P], torch.float32).cpu().numpy()
        ups = crafted_uploads(rng, trainers, P, global_now, rnd)
        byz = (trainers[-1],) if len(trainers) > 1 else ()
        n_samples = {t: 100 + 7 * t for t in trainers}
        correct = {c: rng.integers(0, N_VAL + 1, size=len(trainers)).tolist() for c in comm}
        e = h.round(ups, correct, n_samples, byz)
        errs = h.drain()
        assert errs == [[]] * R, errs                   # every host ledger accepts every record
        blk = h.replicas[0].host_ledger.blocks()[-1]
        assert blk["epoch"] == e and blk["selected"], blk
        sel = blk["selected"]
        vals = np.stack([h.view(t, f"upload_master{e & 1}", [P], torch.float32).cpu().numpy() for t in sel])
        if rule == "fedavg":
            ref = fedavg_reference(vals, blk["weight"])
        else:
            ref = robust_combine(vals, aggregation_trim(rule, trim))
        ref_b16 = torch.from_numpy(ref).to(torch.bfloat16).float().numpy()
        for r in range(R):
            for reg, b16 in (("global", "global_shadow"), ("work_master", "work_shadow")):
                got = h.view(r, reg, [P], torch.float32).cpu().numpy()
                ok = same(got, ref)
                assert ok.all(), (f"round {rnd} rank {r} {reg}: {int((~ok).sum())} coords differ, first "
                                  f"{np.flatnonzero(~ok)[:4]} got {got[~ok][:4]} want {ref[~ok][:4]}")
                gb = h.view(r, b16, [P], torch.bfloat16).float().cpu().numpy()
                assert same(gb, ref_b16).all(), f"round {rnd} rank {r} {b16}: not the RNE of the fp32 result"


@pytest.mark.gpu
def test_harness_robust_rule_bounds_a_byzantine_update():
    """R = 8, every admitted update selected, one byz_mode=1 trainer: median and trimmed mean keep
    every coordinate inside the honest updates' range, FedAvg does not."""
    P, R = 8 * 256, 8
    out = {}
    for rule in ("fedavg", "median", "trimmed_mean"):
        h = ReplicaHarness(R, P, n_comm=2, aggregate_count=6, aggregation=rule, trim=1)
        rng = np.random.default_rng(5)
        g0 = np.zeros(P, np.float32)
        trainers = list(range(2, R))
        ups = {t: torch.from_numpy((g0 + rng.standard_normal(P).astype(np.float32) * 0.01)).cuda() for t in trainers}
        e = h.round(ups, {c: [N_VAL] * 6 for c in (0, 1)}, {t: 100 for t in trainers}, byz=(7,))
        assert h.drain() == [[]] * R
        honest = np.stack([ups[t].cpu().numpy() for t in trainers if t != 7])
        got = h.view(3, "global", [P], torch.float32).cpu().numpy()
        out[rule] = ((got >= honest.min(0)) & (got <= honest.max(0))).all()
        assert e == 0
    assert out["median"] and out["trimmed_mean"] and not out["fedavg"], out


def _solo_cfg(**kw):
    from bflc_demo_b200.config import FLConfig
    return FLConfig.for_world(1, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_fused_engine_solo_robust_rule(dtype):
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine

    # solo: one selected update, which the median returns unchanged (a trimmed mean needs
    # 2 * trim < aggregate_count, i.e. more than one client; the harness covers it)
    cfg = _solo_cfg(hidden=256, batch_size=128, samples_per_client=512, learning_rate=0.01, dtype=dtype,
                    aggregation="median")
    shard = femnist_like(1, 512, seed=3)[0]
    eng = FusedEngine(cfg, shard, rank=0, world=1, device=0)
    eng.capture()
    for _ in range(2):
        st = eng.run_round_e2e()
    assert eng.drain_blocks() == []
    assert st["epoch"] == 3
    torch.cuda.synchronize()
    up = eng.heap.view(eng.layout.offsets[f"upload_master{(st['epoch'] - 1) & 1}"], [eng.n_params], torch.float32)
    assert torch.equal(eng.global_master, up) and torch.equal(eng.work_master, up)


@pytest.mark.gpu
def test_generic_engine_solo_robust_rule():
    from bflc_demo_b200.data.synthetic import cifar_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import LeNet5

    cfg = _solo_cfg(model="lenet5", dataset="cifar10", batch_size=64, samples_per_client=128,
                    learning_rate=0.01, aggregation="median")
    shard = cifar_like(1, 128, seed=3, alpha=0.0)[0]
    eng = GenericFedEngine(cfg, LeNet5(10), shard, rank=0, world=1, device=0)
    eng.capture()
    for _ in range(2):
        st = eng.run_round()
    torch.cuda.synchronize()
    assert eng.drain_blocks() == []
    e = eng.read_state()["epoch"]
    assert e == 3, st
    up = eng.heap.view(eng.layout.offsets[f"upload_master{(e - 1) & 1}"], [eng.n_params], torch.float32)
    assert torch.equal(eng.global_master, up) and torch.equal(eng.work_master, up)


@pytest.mark.gpu
def test_multi_gpu_robust_check():
    n = torch.cuda.device_count()
    if n < 4:
        pytest.skip("needs 4 GPUs")
    n = 8 if n >= 8 else 4
    cmd = [sys.executable, "-m", "torch.distributed.run", f"--nproc_per_node={n}",
           str(ROOT / "scripts" / "multi_gpu_check.py"), "robust"]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1800,
                       env=dict(os.environ, PYTHONPATH=str(ROOT)))
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    line = [ln for ln in p.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    res = json.loads(line[len("RESULT "):])["robust"]
    for name, r in res.items():
        assert r["errs"] == [] and r["identical"] and r["bit_exact"], (name, r)
        if "fedavg" in name:
            assert r["byz_rounds"] > 0 and not r["inside_honest"], (name, r)
        else:
            assert r["inside_honest"], (name, r)
