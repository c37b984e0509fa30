"""Round protocol conformance on one GPU: k_plan, k_upload, first-K admission, k_pull, k_pull_blob,
staged validation and the consensus record of R emulated ranks, each checked against the exact host
models of ``test_protocol_spec_host.py``.

``ProtocolHarness`` extends the replica harness of ``test_gpu_robust_aggregation.py`` with what the
engines pass and that harness does not: plan layers, staged validation (bf16 staging with the fp32
bias ranges, or MXFP8 blobs), first-K admission with a chosen upload order, per-trainer sample /
loss counts, byzantine uploads, ``weight_by_score``, any ``n_val``, and the committee steps
(``fed_pull_candidates``, ``fed_pull_blobs``, ``mlp_val``) on the plan's own ``GemmDynamic``.
Every launch is sequential on one stream, so before each launch that waits the harness asserts on the
host that the flag words and admission slots it polls already hold their targets: a harness bug fails
in Python and never spins on the device.  A committee rank or two-shot slice owner that has not run
yet gets its score row / slice digest written for it, with the exact value its own launch writes
later (score rows only for power-of-two n_val, slice digests from the host reference model)."""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from test_gpu_robust_aggregation import ReplicaHarness, fedavg_reference, same  # noqa: E402
from test_gpu_val_split import w1_map, w2_map  # noqa: E402
from test_protocol_spec_host import (BYZ_SCALES, COMM, E2E, FLAG_DONE, FLAG_SCORED, FLAG_SLICE,  # noqa: E402
                                     FLAG_TRAINED, KMAX, TRAINER, admission, avg_cost_bound, byz_fixture,
                                     byz_upload, digest, exact_mlp, first_k, fp64_predictions, labels_for,
                                     mlp_blob_layout, plan_model, slice_digests, two_shot_slices, unpack_model,
                                     val_inputs)
from test_optim_spec_host import rne_bf16, same_bf16  # noqa: E402

gpu = pytest.mark.gpu
META_CANARY = 0xEEEEEEEE
U16_CANARY, U8_CANARY, F32_CANARY = 0x7FC3, 0xCD, 0x7FC01234


def _np(t):
    return t.cpu().numpy()


class ProtocolHarness(ReplicaHarness):
    """R ranks: ranks [0, n_comm) start as the committee; ``n_needed`` < #trainers is first-K mode."""

    def __init__(self, R, n_params, *, n_comm, aggregate_count, n_needed=None, two_shot=False, extra_bytes=0):
        from bflc_demo_b200._native import ledger
        from bflc_demo_b200.parallel.layout import HeapLayout
        super().__init__(R, n_params, n_comm=n_comm, aggregate_count=aggregate_count, two_shot=two_shot)
        sz, m = self.sz, self.m
        self.layout = HeapLayout(n_params, self.layout.ring_slots, extra_bytes=extra_bytes)
        self.heaps = self.ptrs = None
        self.heaps = [m.SymmHeap(self.layout.total_bytes, 0, 1, 0, "local") for _ in range(R)]
        self.ptrs = [h.local_ptr() for h in self.heaps]
        self.feds = [self.layout.fed_dict(r, R, self.ptrs, 0) for r in range(R)]
        self.lay = dict(self.layout.offsets, n_params=n_params)
        roles = [COMM] * n_comm + [TRAINER] * (R - n_comm)
        self.n_needed = n_needed or (R - n_comm)
        st = m.state_init_bytes(R, n_comm, aggregate_count, roles, self.n_needed)
        L = ledger()
        for r, rep in enumerate(self.replicas):
            self._zero(r)
            self.view(r, "state", [sz["RoundState"]], torch.uint8).copy_(torch.frombuffer(bytearray(st), dtype=torch.uint8))
            self.view(r, "plan", [sz["RoundPlan"]], torch.uint8).fill_(0x5A)
            lc = rep.host_ledger.config()
            lc.needed_update_count = self.n_needed
            rep.host_ledger = L.Ledger(lc)
            rep.host_ledger.Bootstrap(roles)
            rep.state_bytes = self.view(r, "state", [sz["RoundState"]], torch.uint8)
            rep.ring_bytes = self.view(r, "ring", [self.layout.ring_slots * sz["BlockRecord"]], torch.uint8)
        torch.cuda.synchronize()

    def _zero(self, r):
        o, sz, K = self.layout.offsets, self.sz, self.K
        self.flags(r).zero_()
        self.view(r, "admit", [2 * sz["AdmitPage"]], torch.uint8).zero_()
        self.view(r, "scores", [2 * K * K * 4 + 2 * K * 8], torch.uint8).zero_()
        self.view(r, "meta", [2 * K * sz["UploadMeta"]], torch.uint8).zero_()

    # ---------------------------------------------------------------- device words
    def plan_bytes(self, r):
        return self.view(r, "plan", [self.sz["RoundPlan"]], torch.uint8)

    def plan_ptr(self, r):
        return self.ptrs[r] + self.layout.offsets["plan"]

    def read_plan(self, r, n_layers):
        sz = self.sz
        b = _np(self.plan_bytes(r))

        def i32(off, n=1):
            return b[off:off + 4 * n].view(np.int32).tolist()

        def u64(off, n=1):
            return [int(x) for x in b[off:off + 8 * n].view(np.uint64)]
        out = dict(is_trainer=i32(sz["plan_is_trainer_off"])[0], is_comm=i32(sz["plan_is_comm_off"])[0],
                   parity=i32(sz["plan_parity_off"])[0], n_cand=i32(sz["plan_n_cand_off"])[0],
                   cand_rank=i32(sz["plan_cand_rank_off"], KMAX), cand_blob=u64(sz["plan_cand_blob_off"], KMAX),
                   correct=i32(sz["plan_correct_off"], KMAX),
                   loss_sum=float(b[sz["plan_loss_sum_off"]:][:4].view(np.float32)[0]),
                   train_correct=i32(sz["plan_train_correct_off"])[0], opt_step=i32(sz["plan_opt_step_off"])[0],
                   opt_total=i32(sz["plan_opt_total_off"])[0], upload_blocks=i32(sz["plan_upload_blocks_off"])[0],
                   consensus_blocks=i32(sz["plan_consensus_blocks_off"])[0],
                   digest_acc=u64(sz["plan_digest_acc_off"])[0], step_barrier=i32(sz["plan_step_barrier_off"])[0],
                   round_seq=int(b[sz["plan_round_seq_off"]:][:4].view(np.uint32)[0]), dyn=[])
        for li in range(n_layers):
            d0 = sz["plan_dyn_off"] + li * sz["GemmDynamic"]
            out["dyn"].append(dict(active=i32(d0)[0], wait_value=i32(d0 + sz["dyn_wait_value_off"])[0],
                                   map_index=i32(d0 + sz["dyn_map_index_off"], KMAX),
                                   bias=u64(d0 + sz["dyn_bias_off"], KMAX),
                                   wait_flag=u64(d0 + sz["dyn_wait_flag_off"], KMAX)))
        return out

    def admit_words(self, r, par):
        w = _np(self.view(r, "admit", [2 * self.sz["AdmitPage"] // 4], torch.int32)).view(np.uint32)
        base = par * self.sz["AdmitPage"] // 4
        s0 = base + self.sz["admit_slot_off"] // 4
        return int(w[base]), [int(x) for x in w[s0:s0 + KMAX]]

    def meta(self, r, par):
        return _np(self.view(r, "meta", [2 * self.K * 2], torch.int32)).view(np.uint32).reshape(2, self.K, 2)[par]

    def record(self, r, e):
        sz = self.sz
        b = _np(self.view(r, "ring", [self.layout.ring_slots * sz["BlockRecord"]], torch.uint8))
        b = b[(e % self.layout.ring_slots) * sz["BlockRecord"]:][:sz["BlockRecord"]]

        def arr(name, dt, n=KMAX):
            o = sz[f"rec_{name}_off"]
            return b[o:o + np.dtype(dt).itemsize * n].view(dt)
        return dict(epoch=int(b[:4].view(np.uint32)[0]), role_before=arr("role_before", np.uint32).tolist(),
                    score_rows=arr("score_rows", np.float32, KMAX * KMAX).reshape(KMAX, KMAX),
                    scored_mask=arr("scored_mask", np.uint32).tolist(), median=arr("median", np.float32),
                    n_samples=arr("n_samples", np.uint32).tolist(), avg_cost=arr("avg_cost", np.float32),
                    weight=arr("weight", np.float32), admitted_mask=int(arr("admitted_mask", np.uint32, 1)[0]),
                    selected_mask=int(arr("admitted_mask", np.uint32, 2)[1]),
                    weight_by_score=int(arr("weight_by_score", np.uint32, 1)[0]),
                    model_digest=int(arr("model_digest", np.uint64, 1)[0]), seq=int(arr("seq", np.uint32, 1)[0]),
                    agg=int(arr("agg", np.uint32, 1)[0]))

    def state_digest(self, r):
        b = _np(self.view(r, "state", [self.sz["RoundState"]], torch.uint8))
        return int(b[self.sz["state_digest_off"]:][:8].view(np.uint64)[0])

    # ---------------------------------------------------------------- steps
    def plan(self, layers=(), staged=False, steps=3, stage_master=(), blobs=None):
        """k_plan on every rank; returns [(device plan, model plan)] per rank.  stage_master[r]: rank
        r's fp32 staging pointer (0: none); blobs[r]: (stage_blob, blob_bytes, upq_off) or None."""
        e, roles = self.epoch(), self.roles()
        out = []
        for r in range(self.R):
            if e >= 2:
                self._expect(r, [FLAG_DONE + q for q in range(self.R)], e - 1, "fed_plan_round")
            prev = self.read_plan(r, 0)
            sm = stage_master[r] if stage_master else 0
            bl = blobs[r] if blobs else None
            kw = dict(blob_stage_ptr=bl[0], blob_bytes=bl[1], upq_off=list(bl[2])) if bl else {}
            self.m.fed_plan_round(self.feds[r], list(layers), steps, staged, stage_master_ptr=sm, **kw)
            torch.cuda.synchronize()
            want = plan_model(rank=r, roles=roles, epoch=e, n_needed=self.n_needed, layers=layers, staged=staged,
                              bases=self.ptrs, lay=self.lay, steps=steps, prev=prev, stage_master=sm, blobs=bl)
            out.append((self.read_plan(r, len(layers)), want))
        return out

    def upload(self, order, work, n_samples, loss_sum, n_loss_terms, byz=(), byz_scale=5.0):
        """Trainers upload in ``order`` (= ticket order): work_master, the plan's loss_sum, fed_upload."""
        for t in order:
            self.view(t, "work_master", [self.P], torch.float32).copy_(work[t])
            self.plan_bytes(t)[self.sz["plan_loss_sum_off"]:][:4].view(torch.float32).fill_(float(loss_sum[t]))
            self.m.fed_upload(self.feds[t], int(n_samples[t]), int(n_loss_terms[t]), 1 if t in byz else 0, byz_scale)
        torch.cuda.synchronize()

    def slots(self):
        """Trainer of every candidate slot, as the device resolves it (asserting it is resolvable)."""
        e, roles = self.epoch(), self.roles()
        par = e & 1
        if not first_k(roles, self.n_needed):
            return [r for r in range(self.R) if roles[r] & TRAINER]
        out = []
        for z in range(self.n_needed):
            w = self.admit_words(0, par)[1][z]
            assert w >> 8 == e + 1, f"slot {z} not admitted for epoch {e} (harness order bug)"
            out.append(w & 0xFF)
        return out

    def expect_committee_inputs(self, c):
        e, roles = self.epoch(), self.roles()
        sl = self.slots()
        if first_k(roles, self.n_needed):
            words = self.admit_words(c, e & 1)[1]
            low = [z for z in range(self.n_needed) if words[z] >> 8 != e + 1]
            assert not low, f"rank {c}: admission slots {low} not tagged {e + 1} (harness order bug)"
        self._expect(c, [FLAG_TRAINED + t for t in sl], e + 1, "committee pull")
        return sl

    def set_correct(self, c, counts):
        self.plan_bytes(c)[self.sz["plan_correct_off"]:][:4 * len(counts)].view(torch.int32).copy_(
            torch.as_tensor(counts, dtype=torch.int32))

    def consensus(self, n_val, weight_by_score=False, model=None):
        """fed_consensus_aggregate on every rank, committee ranks first.  Score rows of committee ranks
        that have not run yet are written from their plan's counts (needs a power-of-two n_val); in
        two-shot mode the later ranks' slice digests come from ``model`` (the expected new global)."""
        e, roles = self.epoch(), self.roles()
        par, K = e & 1, self.K
        comm = [r for r in range(self.R) if roles[r] & COMM]
        sl = self.slots()
        launch = comm + [r for r in range(self.R) if r not in comm]
        counts = {c: self.read_plan(c, 0)["correct"] for c in comm}
        digs = slice_digests(model, self.R) if self.two_shot else None
        for i, r in enumerate(launch):
            fl = self.flags(r)
            for c in launch[i + 1:]:
                if c in comm:
                    assert n_val & (n_val - 1) == 0, "a later committee row is only known exactly for 2^k n_val"
                    row = self.view(r, "scores", [2 * K * K], torch.float32)[(par * K + c) * K:(par * K + c + 1) * K]
                    for z, t in enumerate(sl):
                        row[t] = float(counts[c][z]) / n_val
                    fl[FLAG_SCORED + c] = e + 1
            if self.two_shot:
                sd = self.view(r, "scores", [2 * K * K + 4 * K], torch.float32)[2 * K * K:].view(torch.int64)
                for q in launch[i + 1:]:
                    sd[par * K + q] = int(np.array(digs[q], dtype=np.uint64).view(np.int64))
                    fl[FLAG_SLICE + q] = e + 1
            self._expect(r, [FLAG_SCORED + c for c in comm if c != r] + [FLAG_TRAINED + t for t in sl],
                         e + 1, "fed_consensus_aggregate")
            if self.two_shot:
                self._expect(r, [FLAG_SLICE + q for q in range(self.R) if q != r], e + 1, "two-shot publish")
            self.m.fed_consensus_aggregate(self.feds[r], n_val, weight_by_score, self.two_shot, False)
            torch.cuda.synchronize()
        return e


# ------------------------------------------------------------------ plan / upload / admission / consensus
def check_plan(got, want):
    for k in ("is_trainer", "is_comm", "parity", "n_cand", "correct", "train_correct", "upload_blocks",
              "consensus_blocks", "digest_acc", "step_barrier", "round_seq", "opt_step", "opt_total", "cand_blob"):
        assert got[k] == want[k], (k, got[k], want[k])
    n = want["n_cand"]
    fk = want["cand_rank"][0] == -1
    assert got["cand_rank"][: KMAX if fk else n] == want["cand_rank"][: KMAX if fk else n]
    assert got["loss_sum"] == 0.0
    for gd, wd in zip(got["dyn"], want["dyn"]):
        assert gd == wd, (gd, wd)


def _work(rng, trainers, P, g):
    return {t: torch.from_numpy((g + rng.standard_normal(P).astype(np.float32) * 0.1).astype(np.float32)).cuda()
            for t in trainers}


PUA = [  # R, n_comm, aggregate_count, n_needed, staged
    pytest.param(4, 1, 3, None, False, id="R4-all-direct"),
    pytest.param(5, 1, 3, None, True, id="R5-all-staged"),
    pytest.param(6, 2, 2, 2, True, id="R6-firstK2-staged"),
    pytest.param(8, 2, 3, 3, True, id="R8-firstK3-staged"),
]


@gpu
@pytest.mark.parametrize("R,n_comm,agg,n_needed,staged", PUA)
def test_plan_upload_admission_and_record(R, n_comm, agg, n_needed, staged):
    """Four rounds with re-election: every rank's plan, every upload byte, meta word, flag, ticket and
    slot word, the committee's untouched buffers, the record and FedAvg over exactly the admitted
    uploads, and the model digest in the record and the ledger page."""
    P = 8 * 1037
    h = ProtocolHarness(R, P, n_comm=n_comm, aggregate_count=agg, n_needed=n_needed)
    rng = np.random.default_rng(R * 10 + (n_needed or 0))
    g0 = (rng.standard_normal(P) * 0.5).astype(np.float32)
    for r in range(R):
        for reg in ("global", "work_master"):
            h.view(r, reg, [P], torch.float32).copy_(torch.from_numpy(g0))
    layers = [(256, True), (4096 + 8, True), (1000, False)]
    stage = [torch.zeros(KMAX, P, device="cuda") for _ in range(R)] if staged else None
    for rnd in range(4):
        e, roles = h.epoch(), h.roles()
        par = e & 1
        trainers = [r for r in range(R) if roles[r] & TRAINER]
        comm = [r for r in range(R) if roles[r] & COMM]
        for got, want in h.plan(layers, staged, steps=3 + rnd,
                                stage_master=[s.data_ptr() for s in stage] if staged else ()):
            check_plan(got, want)
        # canaries: every meta word, the committee's upload buffers
        for r in range(R):
            h.view(r, "meta", [2 * h.K * 2], torch.int32).fill_(int(np.int32(np.uint32(META_CANARY))))
        for c in comm:
            h.view(c, f"upload_master{par}", [P], torch.int32).fill_(int(np.int32(np.uint32(F32_CANARY))))
            h.view(c, f"upload_shadow{par}", [P], torch.int16).fill_(U16_CANARY)
        flags_before = [_np(h.flags(r)).copy() for r in range(R)]
        order = [int(t) for t in rng.permutation(trainers)]
        g_now = _np(h.view(0, "global", [P], torch.float32))
        work = _work(rng, trainers, P, g_now)
        w_spec, g_spec = byz_fixture(P, rnd)
        byz = (order[0],)
        work[order[0]] = torch.from_numpy(w_spec).cuda()
        if len(order) > 1:                                   # an honest upload of the same special values
            work[order[-1]][:36] = torch.from_numpy(w_spec[:36]).cuda()
        for r in range(R):                                   # the byzantine trainer's reference point
            h.view(r, "global", [P], torch.float32)[:64].copy_(torch.from_numpy(g_spec[:64]))
        g_now = _np(h.view(order[0], "global", [P], torch.float32))
        n_samples = {t: 100 + 7 * t + rnd for t in trainers}
        n_terms = {t: (64 if t % 2 else 3 * t + 5) for t in trainers}
        loss = {t: float(np.float32(rng.uniform(0.5, 900.0))) for t in trainers}
        scale = BYZ_SCALES[rnd % 2]
        h.upload(order, work, n_samples, loss, n_terms, byz=byz, byz_scale=scale)
        K = n_needed if first_k(roles, h.n_needed) else len(trainers)
        ticket, slots, admitted = admission(order, K, e)
        fk = first_k(roles, h.n_needed)
        # k_upload: bytes, shadow, meta, flags
        for t in trainers:
            w = _np(work[t])
            want = byz_upload(w, g_now, scale) if t in byz else w
            um = _np(h.view(t, f"upload_master{par}", [P], torch.float32))
            us = _np(h.view(t, f"upload_shadow{par}", [P], torch.int16)).view(np.uint16)
            if t in byz:
                assert same(um, want).all(), np.flatnonzero(~same(um, want))[:5]
            else:
                assert np.array_equal(um.view(np.uint32), want.view(np.uint32))   # bit for bit, NaN payloads too
            assert same_bf16(us, rne_bf16(um)).all(), np.flatnonzero(~same_bf16(us, rne_bf16(um)))[:5]
        for r in range(R):
            meta, fl = h.meta(r, par), _np(h.flags(r))
            for t in range(R):
                if t in admitted:
                    assert int(meta[t, 0]) == n_samples[t]
                    c, b = avg_cost_bound(loss[t], n_terms[t])
                    got = float(meta[t, 1:].view(np.float32)[0])
                    assert abs(got - c) <= b, (t, got, c, b)
                    assert fl[FLAG_TRAINED + t] == e + 1
                else:                                        # committee and late trainers publish nothing
                    assert meta[t].tolist() == [META_CANARY, META_CANARY]
                    assert fl[FLAG_TRAINED + t] == flags_before[r][FLAG_TRAINED + t] <= e
            if fk:
                tw, sw = h.admit_words(r, par)
                assert sw[:K] == [slots[z] for z in range(K)]
                if r == 0:
                    assert tw == ticket
        for c in comm:
            assert (_np(h.view(c, f"upload_master{par}", [P], torch.int32)).view(np.uint32) == F32_CANARY).all()
            assert (_np(h.view(c, f"upload_shadow{par}", [P], torch.int16)).view(np.uint16) == U16_CANARY).all()
        for c in comm:
            h.set_correct(c, rng.integers(0, 65, size=K).tolist())
        h.consensus(64)
        assert h.drain() == [[]] * R
        blk = h.replicas[0].host_ledger.blocks()[-1]
        vals = np.stack([_np(h.view(t, f"upload_master{par}", [P], torch.float32)) for t in blk["selected"]])
        ref = fedavg_reference(vals, blk["weight"])
        for r in range(R):
            rec = h.record(r, e)
            assert rec["admitted_mask"] == sum(1 << t for t in admitted)
            assert set(blk["selected"]) <= set(admitted)
            assert rec["role_before"][:R] == roles and rec["seq"] == e + 1 and rec["agg"] == 0
            assert rec["weight_by_score"] == 0
            for t in admitted:
                assert rec["n_samples"][t] == n_samples[t]
            for c in comm:
                assert rec["scored_mask"][c] == sum(1 << t for t in admitted)
            got = _np(h.view(r, "global", [P], torch.float32))
            assert same(got, ref).all()
            # over the committed bits (a NaN's payload is the device's canonical one)
            assert rec["model_digest"] == digest(got) == h.state_digest(r)


@gpu
def test_ticket_of_a_later_epoch_publishes_nothing():
    """take_ticket == -1: rank 0's ticket word already carries a later round's tag, so every trainer
    writes its upload buffers but publishes no meta, no slot and no flag."""
    R, P = 5, 8 * 256
    h = ProtocolHarness(R, P, n_comm=1, aggregate_count=2, n_needed=2)
    h.plan()
    later = (h.epoch() + 3) << 8
    h.view(0, "admit", [h.sz["AdmitPage"] // 4], torch.int32)[0] = later
    for r in range(R):
        h.view(r, "meta", [2 * h.K * 2], torch.int32).fill_(int(np.int32(np.uint32(META_CANARY))))
    work = {t: torch.full((P,), float(t), device="cuda") for t in range(1, R)}
    h.upload([3, 1, 4, 2], work, {t: 10 for t in work}, {t: 1.0 for t in work}, {t: 1 for t in work})
    for r in range(R):
        assert (_np(h.flags(r))[FLAG_TRAINED:FLAG_TRAINED + KMAX] == 0).all()
        assert (h.meta(r, 0) == META_CANARY).all()
        assert h.admit_words(r, 0)[1] == [0] * KMAX
    assert h.admit_words(0, 0)[0] == later
    for t in work:
        assert bool((h.view(t, "upload_master0", [P], torch.float32) == float(t)).all())


# ------------------------------------------------------------------ k_pull
@gpu
@pytest.mark.parametrize("P", [8 * 1037, 8 * 4096, 8 * 4101], ids=["tail", "unrolled", "unrolled+tail"])
@pytest.mark.parametrize("n_needed", [None, 2], ids=["all", "firstK2"])
def test_pull_candidates(P, n_needed):
    """Slot z of the committee's staging = slot z's trainer's bf16 upload of this parity (ticket order in
    first-K mode), byte for byte; slots >= n_cand and other ranks' staging keep their canaries; the fp32
    master as a full copy and through ranges (coalesced runs, a run at the end, more runs than blocks)."""
    R = 5
    h = ProtocolHarness(R, P, n_comm=1, aggregate_count=2, n_needed=n_needed)
    rng = np.random.default_rng(P + (n_needed or 0))
    nv = P // 4
    ranges = [[0, 1], [1, 2], [7, 3], [nv // 2, 5], [nv // 2 + 9, 1], [nv - 3, 3]]
    for rnd in range(3):
        e, roles = h.epoch(), h.roles()
        par = e & 1
        trainers = [r for r in range(R) if roles[r] & TRAINER]
        comm = [r for r in range(R) if roles[r] & COMM]
        h.plan(staged=True)
        order = [int(t) for t in rng.permutation(trainers)]
        work = {t: torch.from_numpy(rng.standard_normal(P).astype(np.float32)).cuda() for t in trainers}
        h.upload(order, work, {t: 10 + t for t in trainers}, {t: 1.0 for t in trainers}, {t: 1 for t in trainers})
        use_ranges = rnd % 2 == 1
        rt = torch.tensor(ranges, dtype=torch.int64, device="cuda")
        for r in range(R):
            sh = torch.full((KMAX, P), 0, dtype=torch.int16, device="cuda").fill_(U16_CANARY)
            ms = torch.full((KMAX, P), 0, dtype=torch.int32, device="cuda").fill_(F32_CANARY)
            if r in comm:
                sl = h.expect_committee_inputs(r)
            h.m.fed_pull_candidates(h.feds[r], sh, ms.view(torch.float32), rt if use_ranges else None)
            torch.cuda.synchronize()
            shn, msn = _np(sh).view(np.uint16), _np(ms).view(np.uint32)
            if r not in comm:
                assert (shn == U16_CANARY).all() and (msn == F32_CANARY).all()
                continue
            want_order = order[:n_needed] if n_needed else trainers
            assert sl == want_order
            for z in range(KMAX):
                if z >= len(sl):
                    assert (shn[z] == U16_CANARY).all() and (msn[z] == F32_CANARY).all()
                    continue
                t = sl[z]
                up = _np(h.view(t, f"upload_shadow{par}", [P], torch.int16)).view(np.uint16)
                other = _np(h.view(t, f"upload_shadow{1 - par}", [P], torch.int16)).view(np.uint16)
                assert np.array_equal(shn[z], up) and not np.array_equal(up, other)
                um = _np(h.view(t, f"upload_master{par}", [P], torch.int32)).view(np.uint32)
                if not use_ranges:
                    assert np.array_equal(msn[z], um)
                else:
                    mask = np.zeros(P, bool)
                    for o, n in ranges:
                        mask[4 * o:4 * (o + n)] = True
                    assert np.array_equal(msn[z][mask], um[mask]) and (msn[z][~mask] == F32_CANARY).all()
        for c in comm:
            h.set_correct(c, [32] * len(h.slots()))
        h.consensus(64)
        assert h.drain() == [[]] * R


# ------------------------------------------------------------------ k_pull_blob
BLOB_SHAPES = [(784, 256, 62), (64, 256, 10), (112, 128, 1), (1008, 288, 64)]


@gpu
@pytest.mark.parametrize("in_dim,hidden,nc", BLOB_SHAPES, ids=[f"{a}x{b}x{c}" for a, b, c in BLOB_SHAPES])
def test_pull_blobs(in_dim, hidden, nc):
    """Blobs written by quantize_mlp_blob from special_matrix content; slot z in first-K order holds the
    exact dequantised W1 and the first nc rows of W2, and the blob slot b1 | b2; every other byte of
    both slots keeps its canary; both parities."""
    from bflc_demo_b200.models.mlp import mlp_spec
    from bflc_demo_b200.ops.mx8 import quantize_mx8_reference
    from test_gpu_mx8_conformance import special_matrix
    spec = mlp_spec(in_dim, hidden, nc)
    o = {e.name: e.offset for e in spec.entries}
    P = spec.total
    L = mlp_blob_layout(in_dim, hidden)
    from bflc_demo_b200._native import C
    assert C().mx8_mlp_layout(in_dim, hidden) == L
    bb = (L["total"] + 4095) // 4096 * 4096
    R = 4
    h = ProtocolHarness(R, P, n_comm=1, aggregate_count=2, n_needed=2, extra_bytes=2 * bb)
    upq = [h.layout.offsets["extra"], h.layout.offsets["extra"] + bb]
    rng = np.random.default_rng(in_dim + hidden + nc)
    for rnd in range(2):
        e, roles = h.epoch(), h.roles()
        par = e & 1
        trainers = [r for r in range(R) if roles[r] & TRAINER]
        comm = [r for r in range(R) if roles[r] & COMM]
        h.plan(staged=True)
        masters = {}
        for t in trainers:
            m = torch.zeros(P)
            m[:hidden * in_dim] = special_matrix(hidden, in_dim, 10 * rnd + t).clamp(-1e30, 1e30).reshape(-1)
            m[o["b1"]:o["b1"] + hidden] = torch.randn(hidden)
            m[o["w2"]:o["w2"] + nc * hidden] = special_matrix(nc, hidden, 20 + 10 * rnd + t).clamp(-1e30, 1e30).reshape(-1)
            m[o["b2"]:o["b2"] + nc] = torch.randn(nc)
            masters[t] = m
            blob = h.view(t, "extra", [2 * bb], torch.uint8)[par * bb:(par + 1) * bb]
            C().quantize_mlp_blob(m.cuda(), [o["w1"], o["b1"], o["w2"], o["b2"]], in_dim, hidden, nc, blob)
        order = [int(x) for x in rng.permutation(trainers)]
        h.upload(order, {t: masters[t].cuda() for t in trainers}, {t: 5 for t in trainers},
                 {t: 1.0 for t in trainers}, {t: 1 for t in trainers})
        c = comm[0]
        sl = h.expect_committee_inputs(c)
        assert sl == order[:2]
        stage = torch.full((KMAX, bb), U8_CANARY, dtype=torch.uint8, device="cuda")
        dq = torch.full((KMAX, P), 0, dtype=torch.int16, device="cuda").fill_(U16_CANARY)
        C().fed_pull_blobs(h.feds[c], upq[0], upq[1], stage, dq.view(torch.bfloat16), in_dim, hidden, nc,
                           [o["w1"], o["w2"]])
        torch.cuda.synchronize()
        dqn, sn = _np(dq).view(np.uint16), _np(stage)
        for z in range(KMAX):
            if z >= 2:
                assert (dqn[z] == U16_CANARY).all() and (sn[z] == U8_CANARY).all()
                continue
            t = sl[z]
            blob = _np(h.view(t, "extra", [2 * bb], torch.uint8))[par * bb:(par + 1) * bb]
            wdq, wsb = unpack_model(blob, in_dim, hidden, nc, o["w1"], o["w2"], np.full(P, U16_CANARY, np.uint16),
                                    np.full(bb, U8_CANARY, np.uint8))
            assert np.array_equal(dqn[z], wdq), np.flatnonzero(dqn[z] != wdq)[:5]
            assert np.array_equal(sn[z], wsb)
            ref = quantize_mx8_reference(masters[t][:hidden * in_dim].view(hidden, in_dim)).dequantize()
            got = torch.from_numpy(dqn[z][:hidden * in_dim].view(np.int16).copy()).view(torch.bfloat16)
            assert torch.equal(got.float().view(hidden, in_dim), ref)
        h.set_correct(c, [1, 2])
        h.consensus(64)
        assert h.drain() == [[]] * R


# ------------------------------------------------------------------ staged validation end to end
def _e2e(dtype, n_needed):
    from bflc_demo_b200._native import C
    from bflc_demo_b200.engine.base import vector_ranges
    from bflc_demo_b200.models.mlp import mlp_spec
    p = E2E
    in_dim, H, nc, n_val, R = p["in_dim"], p["hidden"], p["nc"], p["n_val"], p["R"]
    spec = mlp_spec(in_dim, H, nc)
    o = {e.name: e.offset for e in spec.entries}
    P = spec.total
    fp8 = dtype == "fp8"
    L = mlp_blob_layout(in_dim, H)
    bb = (L["total"] + 4095) // 4096 * 4096
    h = ProtocolHarness(R, P, n_comm=p["n_comm"], aggregate_count=2, n_needed=n_needed,
                        extra_bytes=2 * bb if fp8 else 0)
    upq = [h.layout.offsets["extra"], h.layout.offsets["extra"] + bb]
    models = {r: exact_mlp(100 + r, in_dim, H, nc, spec) for r in range(R)}
    x = val_inputs(7, n_val, in_dim)
    preds = {r: fp64_predictions(x, models[r], models[r], spec, H, nc) for r in range(R)}
    labels = labels_for(8, [preds[r] for r in range(R)], nc)
    xd = torch.from_numpy(x).to(torch.bfloat16).cuda()
    yd = torch.from_numpy(labels).cuda()
    for r in range(R):                                       # rank 0's stale upload: another model's biases
        for par in (0, 1):
            h.view(r, f"upload_master{par}", [P], torch.float32).copy_(torch.from_numpy(models[r]))
    cand = [torch.zeros(KMAX, P, dtype=torch.bfloat16, device="cuda") for _ in range(R)]
    cmaster = [torch.zeros(KMAX, P, device="cuda") for _ in range(R)]
    cblob = [torch.zeros(KMAX, bb, dtype=torch.uint8, device="cuda") for _ in range(R)]
    ranges = vector_ranges(spec).cuda()
    rng = np.random.default_rng(3)
    report = []
    for rnd in range(2):
        e, roles = h.epoch(), h.roles()
        par = e & 1
        trainers = [r for r in range(R) if roles[r] & TRAINER]
        comm = [r for r in range(R) if roles[r] & COMM]
        h.plan(layers=[(o["b1"], True), (o["b2"], True)], staged=True,
               stage_master=[] if fp8 else [t.data_ptr() for t in cmaster],
               blobs=[(cblob[r].data_ptr(), bb, upq) for r in range(R)] if fp8 else None)
        if fp8:
            for t in trainers:
                blob = h.view(t, "extra", [2 * bb], torch.uint8)[par * bb:(par + 1) * bb]
                C().quantize_mlp_blob(torch.from_numpy(models[t]).cuda(), [o["w1"], o["b1"], o["w2"], o["b2"]],
                                      in_dim, H, nc, blob)
        order = [int(t) for t in rng.permutation(trainers)]
        h.upload(order, {t: torch.from_numpy(models[t]).cuda() for t in trainers}, {t: 50 for t in trainers},
                 {t: 1.0 for t in trainers}, {t: 1 for t in trainers})
        counts = {}
        for c in comm:
            sl = h.expect_committee_inputs(c)
            if fp8:
                C().fed_pull_blobs(h.feds[c], upq[0], upq[1], cblob[c], cand[c], in_dim, H, nc, [o["w1"], o["w2"]])
            else:
                C().fed_pull_candidates(h.feds[c], cand[c], cmaster[c], ranges)
            maps = bytearray(2 * KMAX * 128)
            for z in range(KMAX):
                base = cand[c].data_ptr() + z * P * 2
                maps[z * 128:(z + 1) * 128] = w1_map(base + o["w1"] * 2, in_dim)
                maps[(KMAX + z) * 128:(KMAX + z + 1) * 128] = w2_map(base + o["w2"] * 2, nc)
            mt = torch.frombuffer(maps, dtype=torch.uint8).cuda()
            pp = h.plan_ptr(c)
            corr = h.plan_bytes(c)[h.sz["plan_correct_off"]:][:4 * KMAX].view(torch.int32)
            dyn = [pp + h.sz["plan_dyn_off"] + i * h.sz["GemmDynamic"] for i in range(2)]
            C().mlp_val(xd, yd, corr, mt, dyn[0], dyn[1], n_val, in_dim, H, nc, R,
                        pp + h.sz["plan_cand_blob_off"] if fp8 else 0)
            torch.cuda.synchronize()
            counts[c] = _np(corr).tolist()
            want = [int((preds[t] == labels).sum()) for t in sl]
            report.append((rnd, c, sl, counts[c][:len(sl)], want))
        h.consensus(n_val)
        assert h.drain() == [[]] * R
        rec = h.record(0, e)
        report.append((rnd, "median", sl, [float(rec["median"][t]) for t in sl],
                       [float(np.float32(int((preds[t] == labels).sum()) / n_val)) for t in sl]))
    return report


@gpu
@pytest.mark.parametrize("n_needed", [None, 2], ids=["all", "firstK2"])
@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_staged_validation_end_to_end(dtype, n_needed):
    """plan -> upload -> pull / pull_blob -> mlp_val -> consensus: correct[z], the score rows and the
    record's medians are the fp64 counts of slot z's trainer's own weights and biases."""
    report = _e2e(dtype, n_needed)
    for rnd, c, sl, got, want in report:
        print(f"{dtype} round {rnd} committee {c} slots {sl}: device {got}, fp64 {want}")
    for rnd, c, sl, got, want in report:
        assert got == want, (rnd, c, sl, got, want)


# ------------------------------------------------------------------ consensus record and digests
def _weights_model(n_samples, medians, selected_in_order):
    """run_consensus's weights: w_t = n_t * median_t in fp64, stored as fp32, summed in fp64, w_t / sum."""
    w = {t: float(n_samples[t]) * float(medians[t]) for t in selected_in_order}
    s = 0.0
    for t in selected_in_order:
        s += w[t]
    return {t: np.float32(float(np.float32(w[t])) / s) for t in selected_in_order}


@gpu
def test_consensus_weight_by_score_and_non_power_of_two_n_val():
    """One committee rank (launched first, so no row is pre-written), n_val = 200: score rows within the
    emitted division's bound, weights by score, FedAvg with the record's weights, the record's fields."""
    R, P, n_val = 5, 8 * 517, 200
    h = ProtocolHarness(R, P, n_comm=1, aggregate_count=3)
    rng = np.random.default_rng(9)
    trainers = [1, 2, 3, 4]
    h.plan()
    work = _work(rng, trainers, P, np.zeros(P, np.float32))
    ns = {t: 90 + 11 * t for t in trainers}
    h.upload(trainers, work, ns, {t: 2.0 * t for t in trainers}, {t: 7 for t in trainers})
    counts = [173, 57, 199, 130]
    h.set_correct(0, counts)
    e = h.consensus(n_val, weight_by_score=True)
    assert h.drain() == [[]] * R
    rec = h.record(0, e)
    for z, t in enumerate(trainers):
        c, b = avg_cost_bound(counts[z], n_val)
        assert abs(float(rec["score_rows"][0][t]) - c) <= b
        assert rec["median"][t] == rec["score_rows"][0][t]
    order = sorted(trainers, key=lambda t: -float(rec["median"][t]))[:3]
    wm = _weights_model(ns, {t: rec["median"][t] for t in trainers}, order)
    assert rec["weight_by_score"] == 1 and rec["scored_mask"][0] == 0b11110
    for t in order:
        assert rec["weight"][t] == wm[t], (t, rec["weight"][t], wm[t])
    sel = sorted(order)
    ref = fedavg_reference(np.stack([_np(work[t]) for t in sel]), [rec["weight"][t] for t in sel])
    for r in range(R):
        assert same(_np(h.view(r, "global", [P], torch.float32)), ref).all()
        assert h.record(r, e)["model_digest"] == digest(ref) == h.state_digest(r)


@gpu
@pytest.mark.parametrize("R", [3, 8])
def test_two_shot_every_rank_commits_the_whole_model_digest(R):
    """Two-shot: the later ranks' slice digests are pre-written from the host reference model; every
    rank's record and ledger page must carry the whole-model digest, and every replica the whole model."""
    from bflc_demo_b200.protocol.oracle import run_consensus
    P = 8 * 517
    h = ProtocolHarness(R, P, n_comm=1, aggregate_count=R - 1, two_shot=True)
    rng = np.random.default_rng(R)
    for rnd in range(2):
        e, roles = h.epoch(), h.roles()
        trainers = [r for r in range(R) if roles[r] & TRAINER]
        comm = [r for r in range(R) if roles[r] & COMM]
        h.plan()
        work = _work(rng, trainers, P, _np(h.view(0, "global", [P], torch.float32)))
        ns = {t: 100 + t for t in trainers}
        h.upload(trainers, work, ns, {t: 1.0 for t in trainers}, {t: 1 for t in trainers})
        counts = [int(x) for x in rng.integers(0, 65, len(trainers))]
        h.set_correct(comm[0], counts)
        res = run_consensus(R, 1, R - 1, dict(enumerate(roles)), trainers,
                            {comm[0]: {t: counts[z] / 64 for z, t in enumerate(trainers)}}, ns,
                            {t: 1.0 for t in trainers})
        ref = fedavg_reference(np.stack([_np(work[t]) for t in res.selected]), [res.weight[t] for t in res.selected])
        h.consensus(64, model=ref)
        assert h.drain() == [[]] * R
        assert sum(slice_digests(ref, R)) % (1 << 64) == digest(ref)
        assert all(b > a for a, b in two_shot_slices(P, R)[:-1])
        for r in range(R):
            assert same(_np(h.view(r, "global", [P], torch.float32)), ref).all()
            assert h.record(r, e)["model_digest"] == digest(ref) == h.state_digest(r)
