"""What the two device-protocol engines (``FusedEngine``, ``GenericFedEngine``) share: the genesis roles,
the host views of the device's ``RoundState`` and ``BlockRecord``, and ``ProtocolEngine`` -- the symmetric
heap and its views, the genesis model, the server optimizer and DP state, the ledger page and the host
ledger, the block-ring drain and the consensus launch that closes every round."""
from __future__ import annotations

import struct
from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.distributed as dist

from .._native import C, ledger as _ledger
from ..config import FLConfig
from ..data.synthetic import Shard
from ..parallel.layout import HeapLayout
from ..parallel.symm import SymmetricHeap

ROLE_TRAINER, ROLE_COMM = 1, 2


def step_rows(i: int, batch: int, epoch_rows: int) -> slice:
    """The shard rows local step ``i`` of a round trains on: batch ``i mod E`` of the E = epoch_rows / batch
    whole batches of one local epoch, so epoch k > 0 repeats epoch 0's batches in the same order and no
    step reads past the epoch's rows.  Every engine and ``FlatMLP.train_epoch`` follow this schedule; the
    persistent trainer (mlp_round_sm100.cu) computes the same offset on the device."""
    j = (i % (epoch_rows // batch)) * batch
    return slice(j, j + batch)


def initial_roles(cfg: FLConfig) -> List[int]:
    """Genesis committee (reference: first COMM_COUNT entries in unordered_map order,
    C:176-182 -- arbitrary but deterministic): lowest ids, or a seeded permutation."""
    n = cfg.clients
    if cfg.solo:
        return [ROLE_TRAINER | ROLE_COMM] * n
    ids = list(range(n))
    if cfg.seed:
        rng = np.random.default_rng(cfg.seed)
        rng.shuffle(ids)
    roles = [ROLE_TRAINER] * n
    for i in ids[: cfg.committee_size]:
        roles[i] = ROLE_COMM
    return roles


def resolve_dp_seed(cfg: FLConfig, rank: int, world: int, group) -> int:
    """The DP noise seed every rank uses: cfg.dp_seed, or (None) 64 bits rank 0 draws from ``secrets``
    and broadcasts over the bootstrap group.  0 when no noise is configured (nothing draws from it)."""
    if cfg.dp_mode != 2:
        return 0
    if cfg.dp_seed is not None:
        return int(cfg.dp_seed)
    import secrets
    box = [secrets.randbits(64) if rank == 0 else None]
    if world > 1:
        dist.broadcast_object_list(box, src=0, group=group)
    return int(box[0])


def vector_ranges(spec) -> torch.Tensor:
    """fp32 parts of an update that a forward pass reads from the master copy: every 1-D
    parameter (biases, norm scales / shifts, running statistics); matrices are consumed from
    the bf16 copy.  Coalesced {first float4, float4 count} pairs for ``fed_pull_candidates`` --
    for BERT-base this is 0.1 % of the 437 MB master.  int64 [n, 2] on the CPU."""
    runs = []
    for e in spec.entries:
        if len(e.shape) != 1:
            continue
        lo, hi = e.offset // 4, (e.offset + e.shape[0] + 3) // 4
        if runs and runs[-1][1] >= lo:
            runs[-1][1] = max(runs[-1][1], hi)
        else:
            runs.append([lo, hi])
    return torch.tensor([[lo, hi - lo] for lo, hi in runs], dtype=torch.int64).reshape(-1, 2)


# RoundState (csrc/include/bflc_kernels.h): epoch, n_ranks, n_comm, n_aggregate, role[8],
# last_median[8], selected_mask, global_loss, model_digest, blocks_appended, n_needed
ROUND_STATE = struct.Struct("<4I8I8fIfQII")


def parse_round_state(buf, world: int) -> dict:
    """The ledger page at the start of ``buf`` (a numpy view of the pinned mirror page or of a host copy
    of the device page), cut to ``world`` ranks."""
    f = ROUND_STATE.unpack_from(buf, 0)
    return dict(epoch=f[0], roles=list(f[4:4 + world]), median=list(f[12:12 + world]), selected_mask=f[20],
                global_loss=f[21], model_digest=f[22])


# DpClipRecord (csrc/include/bflc_kernels.h): seq (epoch + 1), clip C_t, noised count b~, n_sel
CLIP_RECORD = struct.Struct("<IffI")
# DpAdapt: clip C_t, quantile, rate, count noise, z_delta, 3 pad words
DP_ADAPT = struct.Struct("<5f3I")


# BlockRecord (csrc/include/bflc_kernels.h), field by field: (name, element count, struct code)
BLOCK_RECORD_FIELDS = (
    ("epoch", 1, "I"), ("n_ranks", 1, "I"), ("n_comm", 1, "I"), ("n_aggregate", 1, "I"),
    ("role_before", 8, "I"), ("role_after", 8, "I"), ("score_rows", 8 * 8, "f"), ("scored_mask", 8, "I"),
    ("median", 8, "f"), ("n_samples", 8, "I"), ("avg_cost", 8, "f"), ("weight", 8, "f"),
    ("admitted_mask", 1, "I"), ("selected_mask", 1, "I"), ("global_loss", 1, "f"), ("weight_by_score", 1, "I"),
    ("model_digest", 1, "Q"), ("seq", 1, "I"), ("agg", 1, "I"))
BLOCK_RECORD = struct.Struct("<" + "".join(f"{n}{code}" for _, n, code in BLOCK_RECORD_FIELDS))


def parse_block_record(buf, offset: int, world: int) -> Tuple[int, int, dict]:
    """The BlockRecord at byte ``offset`` of ``buf``: (its epoch, its seq word, the round as
    ``Ledger.AppendDeviceRound`` takes it, cut to ``world`` ranks)."""
    flat, f, i = BLOCK_RECORD.unpack_from(buf, offset), {}, 0
    for name, n, _ in BLOCK_RECORD_FIELDS:
        f[name] = flat[i] if n == 1 else list(flat[i:i + n])
        i += n
    w = world
    return f["epoch"], f["seq"], dict(
        epoch=f["epoch"], role_before=f["role_before"][:w], role_after=f["role_after"][:w],
        score_rows=[f["score_rows"][8 * c:8 * c + w] for c in range(w)],      # [committee][trainer]
        scored_mask=f["scored_mask"][:w], n_samples=f["n_samples"][:w], avg_cost=f["avg_cost"][:w],
        admitted_mask=f["admitted_mask"], selected_mask=f["selected_mask"], global_loss=f["global_loss"],
        model_digest=f["model_digest"], weight_by_score=f["weight_by_score"], agg=f["agg"])


def drain_ring(host_ledger, ring, drained: int, epoch: int, world: int, clip_ring=None) -> Tuple[int, List[str]]:
    """Append the records of epochs [drained, epoch) out of ``ring`` (a host copy of the device block
    ring) to ``host_ledger``, which re-executes each election.  Stops at the first mismatch.  Returns the
    new drained count and the mismatches ([] = the replicas agree).  ``clip_ring`` (adaptive clipping): a
    host copy of the DpClipRecord ring, whose record of each epoch goes with its block record."""
    rs = BLOCK_RECORD.size
    slots = len(ring) // rs
    errs = []
    while drained < epoch:
        got, seq, rnd = parse_block_record(ring, (drained % slots) * rs, world)
        if got != drained or seq != drained + 1:
            errs.append(f"ring slot for epoch {drained} holds epoch {got} seq {seq}")
            break
        if clip_ring is not None:
            cseq, clip, count, n_sel = CLIP_RECORD.unpack_from(clip_ring, (drained % slots) * CLIP_RECORD.size)
            if cseq != drained + 1:
                errs.append(f"clip record slot for epoch {drained} holds seq {cseq}")
                break
            rnd.update(clip=clip, count=count, n_sel=n_sel)
        msg = host_ledger.AppendDeviceRound(rnd)
        if msg:
            errs.append(f"epoch {drained}: {msg}")
            break
        drained += 1
    return drained, errs


class ProtocolEngine:
    """One rank of the device-resident protocol.  The constructor lays out and fills the symmetric heap
    (genesis model, zeroed server optimizer state and DP page, ledger page) and bootstraps the host
    ledger; a subclass builds its trainer and validation on top and ends every round with
    ``_consensus``.  ``init_(flat, seed=)`` writes the genesis model; ``extra_bytes`` of heap follow the
    standard regions (``layout.offsets["extra"]``)."""

    def __init__(self, cfg: FLConfig, spec, shard: Shard, init_, *, rank: int, world: int, device: int,
                 group, extra_bytes: int = 0):
        self.cfg, self.rank, self.world, self.device, self.group = cfg, rank, world, device, group
        torch.cuda.set_device(device)
        self.dev = torch.device("cuda", device)
        self.mod = C()
        self.sz = sz = self.mod.struct_sizes()
        assert (sz["RoundState"], sz["BlockRecord"]) == (ROUND_STATE.size, BLOCK_RECORD.size), \
            "RoundState / BlockRecord layout changed: update engine/base.py"
        self.spec = spec
        P = self.n_params = spec.total
        B = cfg.batch_size
        self.S = (len(shard) // B) * B  # drop remainder (M:141); the rows of one local epoch
        self.steps = (self.S // B) * cfg.local_epochs    # step i reads step_rows(i, B, S)
        self.n_val = min(cfg.val_samples or len(shard), len(shard))
        # a committee score is hits / validated targets: one per sample for a classifier, one per
        # position for a next-token model (y [n, S])
        self.n_val_targets = int(shard.y[: self.n_val].numel())

        # ---- heap ------------------------------------------------------------------------
        self.layout = HeapLayout(P, cfg.ring_slots, extra_bytes=extra_bytes,
                                 server_state=cfg.server_state_vectors, dp=cfg.dp_mode > 0,
                                 dp_adaptive=cfg.dp_adaptive)
        self.heap = SymmetricHeap(self.layout.total_bytes, rank=rank, world=world, device=device,
                                  group=group, want_multicast=cfg.use_multicast)
        self.fed = self.layout.fed_dict(rank, world, self.heap.peer_ptrs, self.heap.mc_ptr)
        self.multicast = cfg.use_multicast and self.heap.has_multicast
        o, hv = self.layout.offsets, self.heap.view
        self.work_master = hv(o["work_master"], [P], torch.float32)
        self.work_shadow = hv(o["work_shadow"], [P], torch.bfloat16)
        self.global_master = hv(o["global"], [P], torch.float32)
        self.global_shadow = hv(o["global_shadow"], [P], torch.bfloat16)
        self.state_bytes = hv(o["state"], [sz["RoundState"]], torch.uint8)
        self.plan_bytes = hv(o["plan"], [sz["RoundPlan"]], torch.uint8)
        self.ring_bytes = hv(o["ring"], [cfg.ring_slots * sz["BlockRecord"]], torch.uint8)
        self.plan_ptr = self.heap.local_ptr + o["plan"]
        self.loss_sum = hv(o["plan"] + sz["plan_loss_sum_off"], [1], torch.float32)
        self.val_correct = hv(o["plan"] + sz["plan_correct_off"], [sz["kMaxRanks"]], torch.int32)
        self.grad = torch.zeros(P, device=self.dev, dtype=torch.float32)

        # genesis model: identical on every rank
        init = torch.empty(P, dtype=torch.float32)
        init_(init, seed=cfg.seed + 1234)
        for t in (self.work_master, self.global_master):
            t.copy_(init)
        for t in (self.work_shadow, self.global_shadow):
            t.copy_(init.to(torch.bfloat16))
        # server optimizer state (this rank's own; m = v = 0 at genesis)
        self.server_state = [hv(o[k], [P], torch.float32) for k in ("server_m", "server_v")[: cfg.server_state_vectors]]
        for t in self.server_state:
            t.zero_()
        self.server_kw = self.layout.server_opt_kwargs(cfg.server_opt_id, cfg.server_opt_constants)
        # differential privacy: the noise seed (resolved once, the same on every rank), the consensus
        # kernel's DP arguments and a zeroed DpPage (its block ticket must start at 0)
        self.dp_seed = resolve_dp_seed(cfg, rank, world, group)
        clip, noise = cfg.dp_constants
        self.dp_kw = self.layout.dp_kwargs(cfg.dp_mode, clip, noise, self.dp_seed, cfg.dp_adaptive)
        self.dp_page = hv(o["dp"], [sz["DpPage"]], torch.uint8) if cfg.dp_mode > 0 else None
        if self.dp_page is not None:
            self.dp_page.zero_()
        # adaptive clipping: the DpAdapt header (C_0 and the constants) and a zeroed clip-record ring
        self.dp_adapt = self.clip_ring = None
        if cfg.dp_adaptive:
            head, ring = self.layout.dp_adapt_offsets()
            q, lr, sb = cfg.dp_adapt_constants
            self.dp_adapt = hv(head, [sz["DpAdapt"]], torch.uint8)
            self.dp_adapt.copy_(torch.frombuffer(bytearray(self.mod.dp_adapt_bytes(
                float(clip), float(noise), float(q), float(lr), float(sb))), dtype=torch.uint8))
            self.clip_ring = hv(ring, [cfg.ring_slots * sz["DpClipRecord"]], torch.uint8)
            self.clip_ring.zero_()

        # ledger page + host chain
        roles = initial_roles(cfg)
        st = self.mod.state_init_bytes(world, cfg.committee_size, cfg.aggregate_count, roles,
                                       cfg.needed_updates)
        self.state_bytes.copy_(torch.frombuffer(bytearray(st), dtype=torch.uint8))
        self.host_ledger = _ledger().Ledger(self.ledger_config())
        self.host_ledger.Bootstrap(roles)
        self.drained = 0
        self._rounds = 0
        self._drain_every = max(cfg.ring_slots // 2, 1)

        self.byz = 1 if rank in cfg.byzantine_ranks else 0
        self.straggle_us = cfg.straggler_delay_us if rank in cfg.straggler_ranks else 0
        self.staged = bool(cfg.stage_candidates) and world > 1

    # ------------------------------------------------------------------ one round
    def _next_round(self):
        """Count the round about to be launched.  The consensus kernel writes epoch e's BlockRecord into
        ring slot e % ring_slots: drain the ring into the host ledger before a slot can be overwritten."""
        self._rounds += 1
        if self._rounds - self.drained >= self._drain_every:
            errs = self.drain_blocks()
            if errs:
                raise RuntimeError(f"host/device ledgers disagree: {errs[:2]}")

    def _consensus(self, mirror_ptr: int = 0, seq_ptr: int = 0):
        """UploadScores + Aggregate + QueryGlobalModel (with DP: every update's norm first).  ``mirror_ptr``:
        pinned page the committed ledger page is mirrored into; ``seq_ptr``: fed-rounds word to bump."""
        m, cfg = self.mod, self.cfg
        if self.dp_kw:
            m.fed_update_norms(self.fed, self.layout.offsets["dp"])
        m.fed_consensus_aggregate(self.fed, self.n_val_targets, cfg.weight_by_score, self.two_shot, self.multicast,
                                  mirror_ptr, seq_ptr, cfg.aggregation_rule, cfg.trim,
                                  **self.server_kw, **self.dp_kw)

    @property
    def consensus_captured(self) -> bool:
        """Whether the consensus launch, DP seed included, is baked into a captured graph (then a
        checkpoint's DP seed can no longer be adopted)."""
        return False

    # ------------------------------------------------------------------ host views
    def read_state(self, buf: Optional[torch.Tensor] = None) -> dict:
        """The ledger page: a synchronous copy of the device's, or the host copy in ``buf``."""
        return parse_round_state((self.state_bytes.cpu() if buf is None else buf).numpy(), self.world)

    def drain_blocks(self) -> List[str]:
        """Pull finished BlockRecords off the device ring into the host C++ ledger, which
        re-executes each election.  Returns the list of mismatches ([] = replicas agree)."""
        torch.cuda.synchronize()
        epoch = self.read_state()["epoch"]
        self.drained, errs = drain_ring(self.host_ledger, self.ring_bytes.cpu().numpy(), self.drained, epoch,
                                        self.world, None if self.clip_ring is None else self.clip_ring.cpu().numpy())
        return errs

    def read_stamps(self) -> dict:
        """%globaltimer phase stamps (ns) of the LAST finished round on this rank, turned into
        durations (us).  ``exposed_comm_us`` = upload + candidate pull + consensus/FedAvg/publish,
        i.e. everything in the round that is neither local training nor the validation GEMMs."""
        torch.cuda.synchronize()
        raw = bytes(self.plan_bytes.cpu().numpy())
        t = struct.unpack_from("<8Q", raw, self.sz["plan_stamps_off"])

        def d(a, b):
            return (t[b] - t[a]) / 1e3 if t[a] and t[b] and t[b] >= t[a] else 0.0
        out = dict(train_us=d(0, 1) if t[1] else 0.0, upload_us=d(1, 2), pull_us=d(3, 4),
                   # direct (unstaged) validation has no pull stamps: it starts after the upload
                   validate_us=d(4, 5) if t[4] else (d(2, 5) if t[2] else 0.0),
                   consensus_wait_us=d(5, 6),
                   aggregate_publish_us=d(6, 7), round_us=d(0, 7))
        # pull_us on a committee rank includes waiting for the trainers' flags (it starts with
        # the round); the exposed part is what is left of the round after compute
        out["exposed_comm_us"] = max(out["round_us"] - out["train_us"] - out["validate_us"], 0.0)
        return out

    def ledger_config(self):
        """The host ledger's configuration: the engine's config with the resolved DP seed."""
        lc = self.cfg.to_ledger_config(self.n_params)
        lc.dp_seed = self.dp_seed
        return lc

    def last_update_norms(self, with_clip: bool = False):
        """L2 norms of the last committed round's update model changes (upload - global), by trainer
        rank, float32 [world], NaN for a rank whose update was not admitted; None with DP off.
        ``with_clip``: (norms, C_t, b~) -- also the clip that round used and its noised count of unclipped
        selected updates (adaptive clipping; with a fixed clip C_t is dp_clip and b~ None)."""
        if self.dp_page is None:
            return None
        torch.cuda.synchronize()
        off = self.sz["dp_norm_off"]
        norms = self.dp_page[off:off + 4 * self.world].cpu().numpy().view(np.float32).copy()
        if not with_clip:
            return norms
        if self.clip_ring is None:
            return norms, np.float32(self.cfg.dp_constants[0]), None
        e = self.read_state()["epoch"]
        if e == 0:
            return norms, np.float32(self.clip_now()), None
        _, clip, count, _ = CLIP_RECORD.unpack_from(self.clip_ring.cpu().numpy(),
                                                    ((e - 1) % self.cfg.ring_slots) * CLIP_RECORD.size)
        return norms, np.float32(clip), np.float32(count)

    def clip_now(self) -> float:
        """The clip the next round uses (adaptive clipping: C_t from the device's DpAdapt header)."""
        if self.dp_adapt is None:
            return float(self.cfg.dp_constants[0])
        torch.cuda.synchronize()
        return DP_ADAPT.unpack(bytes(self.dp_adapt.cpu().numpy()))[0]

    def set_clip_now(self, clip: float):
        """Write C_t into the device's DpAdapt header (checkpoint restore)."""
        raw = bytearray(bytes(self.dp_adapt.cpu().numpy()))
        struct.pack_into("<f", raw, 0, float(clip))
        self.dp_adapt.copy_(torch.frombuffer(raw, dtype=torch.uint8))

    def privacy_spent(self) -> tuple:
        """(epsilon, delta) of the committed rounds (protocol/privacy.py): every committed round counts as
        a noised one (a round that selected nothing released nothing new, so this over-counts safely).
        (inf, delta) without noise."""
        from ..protocol.privacy import epsilon
        if self.cfg.dp_mode != 2:
            return float("inf"), self.cfg.dp_delta
        rounds = int(self.read_state()["epoch"])
        return epsilon(float(self.cfg.dp_constants[1]), rounds, self.cfg.dp_delta), self.cfg.dp_delta
