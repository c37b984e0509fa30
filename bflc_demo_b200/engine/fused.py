"""The H100-native round engine: one process per GPU, every rank replays the SAME captured
CUDA graph each round; who trains and who validates is decided by data in the HBM ledger
page (role bits), not by launch topology.

  round graph (all ranks; 7-8 launches):
    fed_plan_round  ||  prep_inputs    QueryState (local read of the ledger page); this round's
                                       inputs (u8 -> bf16, + the dequantised MXFP8 x in fp8 mode) and
                                       the MXFP8 copy of the new global weights on a parallel branch
    [trainer]  mlp_round               the whole local epoch in ONE persistent kernel whose last
                                       optimizer epilogue IS UploadLocalUpdate (writes the upload
                                       buffers, releases FLAG_TRAINED on every peer)
                                       (csrc/kernels/mlp_round_sm100.cu; per-GEMM launches +
                                       fed_upload with ``fused_step=False``: models/mlp.py)
    [committee] fed_pull_*             QueryAllUpdates: each candidate's weights cross NVLink once
                                       (fp8: one 227 KB blob per candidate, unpacked into exact bf16
                                       weights)
                mlp_val                validation of every candidate in one launch (other shapes than
                                       hidden 256 / <= 64 classes: two grouped GEMMs)
    fed_consensus_aggregate            UploadScores + Aggregate + QueryGlobalModel

``cfg.dtype``: "bf16", or "fp8" = BASELINE.json config #2: fwd1/fwd2 of training and the whole
committee validation multiply block-scaled fp8 (MXFP8: e4m3 with UE8M0 block scales) operands,
gradients bf16, master weights / Adam moments fp32.  Hopper has no block-scaled MMA, so every
one of those GEMMs runs as a bf16 wgmma with fp32 accumulation on exactly dequantised copies of
the MXFP8 operands (x_dq, the trainer's work_dq / h_dq, the candidates' dequantised uploads) --
the sum a block-scaled instruction forms (DESIGN.md section 3).

No NCCL call and no host synchronisation inside a round.  The host C++ ledger drains the
device block ring afterwards and re-executes every election (``Ledger.AppendDeviceRound``).

Reference call stacks replaced: SURVEY.md 3.2 (trainer round) and 3.3 (committee round),
i.e. python-sdk/main.py:103-169, 196-228 and CommitteePrecompiled.cpp:215-456.
"""
from __future__ import annotations

import os
import time
import weakref
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from .._native import C
from ..config import FLConfig
from ..data.synthetic import Shard
from ..models.mlp import CHAIN_CLASSES, FlatMLP, check_chain_shapes, mlp_spec
from ..ops import gemm as G
from .base import ROUND_STATE as _ROUND_STATE  # noqa: F401  (the mirror page's layout, importable from here)
from .base import ProtocolEngine, parse_round_state, vector_ranges
from .generic import dpsgd_epsilon, resolve_dpsgd_seed


class FusedDpsgd:
    """The persistent trainer's DP-SGD state where run summaries and checkpoints read it, as they read
    ``ops.dpsgd.DPSGDStep``: this rank's noise key ``seed`` (set it before ``capture``: the round graph
    holds it) and the ``dropped`` counter of examples with a non-finite bound."""

    def __init__(self, trainer: FlatMLP):
        self.trainer = trainer

    @property
    def seed(self) -> int:
        return self.trainer.dpsgd_seed

    @seed.setter
    def seed(self, seed: int):
        self.trainer.dpsgd_seed = int(seed) % (1 << 64)

    @property
    def dropped(self) -> torch.Tensor:
        return self.trainer.dpsgd_dropped


class FusedEngine(ProtocolEngine):
    def __init__(self, cfg: FLConfig, shard: Shard, *, rank: int = 0, world: int = 1,
                 device: int = 0, group=None, in_dim: Optional[int] = None):
        assert cfg.clients == world, "one client per rank"
        assert world <= 8
        if cfg.lora_rank:
            raise ValueError("FusedEngine trains the MLP in full: LoRA (lora_rank > 0) needs GenericFedEngine "
                             "with a bert or gpt LoRANet")
        if cfg.has_optim_recipe:
            raise ValueError("FusedEngine's persistent trainer has no weight decay, lr schedule or gradient "
                             "clipping: run the model through GenericFedEngine for the optimizer recipe")
        if cfg.dpsgd_on and not cfg.dpsgd_fused:
            raise ValueError("FusedEngine's persistent trainer has no per-example clipping: run DP-SGD "
                             "(dpsgd_clip > 0) through GenericFedEngine, or opt in with dpsgd_fused")
        if cfg.dpsgd_fused:
            cfg.validate()

        # ---- model + heap --------------------------------------------------------------
        x0 = shard.x.reshape(len(shard), -1)
        self.in_dim = in_dim or x0.shape[1]
        spec = mlp_spec(self.in_dim, cfg.hidden, shard.n_classes)
        # block-scaled fp8: needs the persistent trainer's shape family (hidden 256, 57..64 classes)
        self.fp8 = cfg.dtype == "fp8"
        if self.fp8 and not (cfg.hidden == 256 and shard.n_classes in CHAIN_CLASSES and cfg.fused_step
                             and cfg.batch_size % 128 == 0 and self.in_dim % 16 == 0
                             and len(shard) % 128 == 0):
            raise ValueError("dtype='fp8' (MXFP8) needs hidden == 256, 57..64 classes, batch % 128 == 0, "
                             "in_dim % 16 == 0, shard rows % 128 == 0 and the fused step")
        # DP-SGD / fp8 shapes the trainer's launcher refuses: here, before the heap or any launch
        check_chain_shapes(self.in_dim, cfg.hidden, shard.n_classes, cfg.batch_size, fp8=self.fp8,
                           dpsgd=cfg.dpsgd_on, prox=cfg.prox_mu > 0, device=device)
        self.ql = C().mx8_mlp_layout(self.in_dim, cfg.hidden) if self.fp8 else None
        self.blob_bytes = (self.ql["total"] + 4095) // 4096 * 4096 if self.fp8 else 0
        super().__init__(cfg, spec, shard, spec.init_, rank=rank, world=world, device=device, group=group,
                         extra_bytes=2 * self.blob_bytes)
        sz, o, hv, P = self.sz, self.layout.offsets, self.heap.view, self.n_params
        plan_ptr = self.plan_ptr
        self.is_trainer_ptr = plan_ptr + sz["plan_is_trainer_off"]
        self.is_comm_ptr = plan_ptr + sz["plan_is_comm_off"]
        self.train_correct = hv(o["plan"] + sz["plan_train_correct_off"], [1], torch.int32)

        # ---- model trainer over heap views -----------------------------------------------
        self.trainer = FlatMLP(self.spec, self.work_master, self.work_shadow, self.grad,
                               cfg.batch_size, optimizer=cfg.optimizer, lr=cfg.learning_rate,
                               loss_sum=self.loss_sum, correct=self.train_correct,
                               step_dev_ptr=plan_ptr + sz["plan_opt_step_off"], fp8=self.fp8,
                               prox_mu=cfg.prox_mu, anchor=self.global_master,
                               **self._dpsgd_kwargs(cfg, rank))
        # DP-SGD (cfg.dpsgd_fused): the trainer clips and noises every local step with this rank's own key
        self.dpsgd = FusedDpsgd(self.trainer) if cfg.dpsgd_on else None
        # upload buffers start as the genesis model (the fused upload never touches the padding
        # elements between tensors; FedAvg must not sum garbage there)
        for par in (0, 1):
            hv(o[f"upload_master{par}"], [P], torch.float32).copy_(self.global_master)
            hv(o[f"upload_shadow{par}"], [P], torch.bfloat16).copy_(self.global_shadow)
        self.upq_off = [o["extra"], o["extra"] + self.blob_bytes] if self.fp8 else []
        if self.fp8:
            for off in self.upq_off:
                self.trainer.quantize_weights(self.global_master, hv(off, [self.blob_bytes], torch.uint8))
            self.trainer.quantize_weights()

        # ---- data ------------------------------------------------------------------------
        self.x_u8 = torch.empty(len(shard), self.in_dim, device=self.dev, dtype=torch.uint8)
        self.x_bf = torch.empty(len(shard), self.in_dim, device=self.dev, dtype=torch.bfloat16)
        # fp8: x's MXFP8 values dequantised (exact in bf16), the fwd1 operand of training and
        # validation; the e4m3 bytes themselves are not needed by anything
        self.x_dq = (torch.empty(len(shard), self.in_dim, device=self.dev, dtype=torch.bfloat16)
                     if self.fp8 else None)
        self.y = torch.empty(len(shard), device=self.dev, dtype=torch.int32)
        self.host_x = x0.contiguous().pin_memory()
        self.host_y = shard.y.to(torch.int32).contiguous().pin_memory()
        self.x_u8.copy_(self.host_x)
        self.y.copy_(self.host_y)
        self.h_val = torch.empty(world, self.n_val, cfg.hidden, device=self.dev, dtype=torch.bfloat16)
        self.out_host = torch.empty(sz["RoundState"], dtype=torch.uint8).pin_memory()

        # ---- validation tensor-map table [layer][parity][rank] (peers' upload shadows) ----
        K = sz["kMaxRanks"]
        e1, e2 = self.spec.by_name["w1"], self.spec.by_name["w2"]
        # N-tile widths are pinned so the pre-encoded peer tensor maps match the launches
        self.val_bn = [self.mod.gemm_pick_bn(e1.shape[0], G.EPI_GENERIC, self.n_val, world),
                       self.mod.gemm_pick_bn(e2.shape[0], G.EPI_ARGMAX, self.n_val, world)]
        # hidden == 256: the whole validation forward of every candidate is ONE launch
        # (mlp_val_sm100: fwd1 -> relu -> fwd2 -> argmax, hidden activations stay in registers /
        # smem).  Each CTA of its 2-CTA clusters computes 128 hidden units: layer-1 maps with a
        # 128-row box.
        self.val_chain = cfg.hidden == 256 and e2.shape[0] <= 64
        if self.val_chain:
            self.val_bn = [128, 64]
        # Two ways to feed the candidates' weights to the validation GEMMs (``self.staged``):
        #  staged (default): fed_pull_candidates streams each trainer's bf16 weights out of its
        #    HBM once (as soon as that trainer's flag is up); the GEMM B maps cover the local
        #    staging slots [layer][slot].
        #  direct: the B maps cover the trainers' upload buffers [layer][parity][rank] and the
        #    GEMM's TMA producer pulls tiles across NVLink itself -- no staging pass, but every
        #    M-tile CTA re-reads the weights remotely (good only for few M-tiles).
        # first-K-wins admission (needed_updates < trainers): candidate slots are resolved on the
        # device from the admission tickets, which needs the staged (pull) validation path
        self.first_k = (not cfg.solo) and cfg.needed_updates < cfg.n_trainers
        if self.first_k and not self.staged:
            raise ValueError("needed_updates < trainers (first-K-wins admission) needs stage_candidates=True")
        # staging slots: bf16 weights in the flat parameter layout (fp8: the blobs unpacked,
        # exactly dequantised), and in fp8 mode a blob-layout slot per candidate of which only
        # the fp32 biases are written
        self.cand_shadow = torch.zeros(world, P, device=self.dev, dtype=torch.bfloat16)
        self.cand_q = (torch.zeros(world, self.blob_bytes, device=self.dev, dtype=torch.uint8)
                       if self.fp8 else None)
        # staged bf16: each candidate's fp32 biases are pulled with its weights into a local fp32 slot,
        # and the plan points slot z's validation biases there -- never at a peer's upload buffer,
        # whose rank the plan does not know in first-K mode (fp8 reads them from the staged blob)
        self.cand_master = self.cand_ranges = None
        if self.staged and not self.fp8:
            self.cand_master = torch.zeros(world, P, device=self.dev, dtype=torch.float32)
            self.cand_ranges = vector_ranges(self.spec).to(self.dev)
        blob = bytearray(2 * 2 * K * 128)

        def b_map(base, e, kind, layer):
            return self.mod.gemm_b_map(base + e.offset * 2, e.shape[0], e.shape[1], e.shape[1], False,
                                       False, kind, self.val_bn[layer])

        for layer, (e, kind) in enumerate(((e1, G.EPI_GENERIC), (e2, G.EPI_ARGMAX))):
            if self.staged:
                for zslot in range(world):
                    base = self.cand_shadow.data_ptr() + zslot * P * 2
                    idx = layer * K + zslot
                    blob[idx * 128:(idx + 1) * 128] = b_map(base, e, kind, layer)
                continue
            for par in range(2):
                for r in range(world):
                    # fp8: the trainer's last optimizer epilogue writes the dequantised blob here
                    base = self.heap.peer_ptrs[r] + o[f"upload_shadow{par}"]
                    idx = (layer * 2 + par) * K + r
                    blob[idx * 128:(idx + 1) * 128] = b_map(base, e, kind, layer)
        self.b_maps = torch.frombuffer(blob, dtype=torch.uint8).to(self.dev)
        self._w_offs = [e1.offset, e2.offset]
        self.plan_layers = [(self.spec.offset("b1"), True), (self.spec.offset("b2"), True)]
        self.dyn_ptr = [plan_ptr + sz["plan_dyn_off"] + i * sz["GemmDynamic"] for i in range(2)]
        # FedAvg as "every rank reduces everything" (one-shot) or "reduce my 1/n slice, publish it
        # to all replicas" (two-shot).  Measured on the 0.87 MB model: two-shot 3301 vs 2988
        # rounds/s at 8 GPUs (8 ranks each pulling 4 whole uploads contend with the committee's
        # pulls), 3612 vs 3671 at 4 GPUs -> two-shot from 8 ranks up, and always for big models.
        self.two_shot = (cfg.two_shot if cfg.two_shot is not None
                         else world > 1 and (P * 4 > (64 << 20) or world >= 8))
        self.fused_step = bool(cfg.fused_step) and self.trainer.fused_ok(self.steps)
        # UploadLocalUpdate inside the trainer's last optimizer epilogue (needs E_OPT)
        self.fused_upload = self.fused_step and os.environ.get("BFLC_MLP_EPIOPT", "1") != "0"
        if self.fp8 and not (self.fused_step and self.fused_upload):
            raise ValueError("dtype='fp8' needs the persistent trainer with the optimizer epilogue")
        if self.dpsgd is not None and not (self.fused_step and self.fused_upload):
            raise ValueError("dpsgd_fused needs the persistent trainer (within its shape limits) with the "
                             "optimizer epilogue")
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.graph_pipe: Optional[torch.cuda.CUDAGraph] = None
        self._exec: Dict[int, int] = {}
        self.stream = torch.cuda.Stream(device=self.dev)
        self._side = torch.cuda.Stream(device=self.dev)
        self._side2 = torch.cuda.Stream(device=self.dev)
        self._ev_fork, self._ev_join = torch.cuda.Event(), torch.cuda.Event()
        # host -> device input pipeline (run_round_e2e): needs the one-launch trainer (its producer
        # waits per step) and a shard of exactly E whole batches, E <= 16 (one chunk and one flag word
        # of in_flags / x_ready per batch of the epoch; later local epochs reread the same chunks)
        self.epoch_steps = self.S // cfg.batch_size
        self.pipelined_input = (self.fused_step and self.S == len(shard) and self.epoch_steps <= 16
                                and (cfg.batch_size * self.in_dim) % 16 == 0
                                and os.environ.get("BFLC_INPUT_PIPELINE", "1") != "0"
                                and os.environ.get("BFLC_MLP_CHAIN", "3") != "1")
        # result read-back of run_round_e2e: the consensus kernel mirrors the committed ledger page
        # into this pinned page and release-stores the new epoch into word MIRROR_SEQ; the host
        # polls it (no copy-engine launch, no stream sync at the end of a round)
        self.mirror = torch.zeros(128, dtype=torch.int32).pin_memory()
        self._mirror_np = self.mirror.numpy()
        self._epoch_known: Optional[int] = None
        self.mirror_result = os.environ.get("BFLC_RESULT_MIRROR", "1") != "0"
        self.in_flags = torch.zeros(16, device=self.dev, dtype=torch.int32)
        self.in_seq = torch.zeros(1, device=self.dev, dtype=torch.int32)
        self.cast_cnt = torch.zeros(16, device=self.dev, dtype=torch.int32)
        self.x_ready = torch.zeros(16, device=self.dev, dtype=torch.int32)
        self.in_err = torch.zeros(1, device=self.dev, dtype=torch.int32)
        self._ev_wq = torch.cuda.Event()
        self.seq_host = torch.zeros(1, dtype=torch.int32).pin_memory()
        self._seq_np = self.seq_host.numpy()
        self._seq = 0
        self._copy_stream = torch.cuda.Stream(device=self.dev)
        # constant arguments of the per-round h2d_pipeline call (kept off the per-round Python path)
        self._pipe_dst, self._pipe_y = self.x_u8.data_ptr(), self.y.data_ptr()
        self._pipe_chunk = self.cfg.batch_size * self.in_dim
        self._pipe_flags = (self.in_flags.data_ptr(), self.seq_host.data_ptr(), self._copy_stream.cuda_stream)
        self._prefeed = os.environ.get("BFLC_E2E_PREFEED", "1") == "1"
        self._host_checked: Dict[int, weakref.ref] = {}     # id -> host input tensor already checked
        self._tag_wv = os.environ.get("BFLC_E2E_TAGS", "writevalue") != "memcpy"
        self.launches_per_round = 0
        if world > 1:
            dist.barrier(group=group)
        torch.cuda.synchronize()

    # ------------------------------------------------------------------ one round
    def _enqueue_round(self, pipe: bool = False):
        """One round.  ``pipe``: the input-pipeline variant used by ``run_round_e2e`` (chunked,
        tag-driven input conversion overlapping the training steps); the plain variant converts
        the resident inputs up front.  Both leave identical state."""
        m, cfg = self.mod, self.cfg
        pipe = pipe and self.pipelined_input
        n0 = m.launch_count()
        # The input cast does not depend on the plan: it runs as a parallel branch of the captured
        # graph.  With the input pipeline it is a persistent kernel that converts chunk s (the rows
        # of local step s) as soon as that chunk's H2D copy has landed (run_round_e2e), and the
        # trainer's TMA producer waits per step -- the branch is joined only before validation.
        main = torch.cuda.current_stream()
        self._ev_fork.record(main)
        self._side.wait_event(self._ev_fork)
        B = cfg.batch_size
        if self.fp8:
            # the consensus kernel of the previous round rewrote the training weights: refresh this
            # trainer's MXFP8 copy (e4m3 + scale chunks) before step 0 -- a third parallel branch
            self._side2.wait_event(self._ev_fork)
            with torch.cuda.stream(self._side2):
                self.trainer.quantize_weights()
                self._ev_wq.record(self._side2)
        with torch.cuda.stream(self._side):
            if pipe:
                m.prep_inputs_chunks(self.x_u8, self.x_bf, None, None, B, self.epoch_steps,
                                     1.0 / 255.0, self.in_flags, self.in_seq, self.cast_cnt,
                                     self.x_ready, self.in_err, self.x_dq)
            else:
                m.prep_inputs(self.x_u8, self.x_bf, None, None, 1.0 / 255.0, self.x_dq)
            self._ev_join.record(self._side)
        if self.fp8:
            m.fed_plan_round(self.fed, self.plan_layers, self.steps, self.staged,
                             self.cand_q.data_ptr(), self.blob_bytes, self.upq_off)
        else:
            m.fed_plan_round(self.fed, self.plan_layers, self.steps, self.staged,
                             stage_master_ptr=self.cand_master.data_ptr() if self.cand_master is not None else 0)
        if not pipe:
            main.wait_event(self._ev_join)
        if self.fp8:
            main.wait_event(self._ev_wq)
        # local training, predicated on the trainer role bit
        m.set_predicate(self.is_trainer_ptr)
        if self.fused_step:
            # every local step of the round inside ONE persistent kernel (phase barriers instead
            # of launches); the barrier word lives in the plan and is zeroed by k_plan.  With
            # fused_upload its last optimizer epilogue publishes the update (UploadLocalUpdate).
            up = dict(fed=self.fed, upq_off=self.upq_off, n_samples=self.S,
                      n_loss_terms=self.steps * B, byz_mode=self.byz,
                      byz_scale=cfg.byzantine_scale, straggle_us=self.straggle_us) if self.fused_upload else {}
            self.trainer.train_epoch_fused(
                self.x_bf, self.y, self.steps, self.plan_ptr + self.sz["plan_step_barrier_off"],
                None, -1, -1,
                self.x_ready.data_ptr() if pipe else 0, self.in_seq.data_ptr() if pipe else 0,
                x_dq=self.x_dq, epoch_rows=self.S, **up)
        else:
            self.trainer.train_epoch(self.x_bf, self.y, self.steps, epoch_rows=self.S)
        m.set_predicate(0)
        if pipe:
            main.wait_event(self._ev_join)      # validation reads every converted row
        if not (self.fused_step and self.fused_upload):
            m.fed_upload(self.fed, self.S, self.steps * B, self.byz, cfg.byzantine_scale, self.straggle_us)
        # committee validation: grouped GEMMs whose B operands are the trainers' uploads
        if self.staged:
            if self.fp8:
                m.fed_pull_blobs(self.fed, self.upq_off[0], self.upq_off[1], self.cand_q, self.cand_shadow,
                                 self.in_dim, cfg.hidden, self.spec.by_name["w2"].shape[0], self._w_offs)
            else:
                m.fed_pull_candidates(self.fed, self.cand_shadow, self.cand_master, self.cand_ranges)
        H = cfg.hidden
        yv = self.y[: self.n_val]
        if self.val_chain:
            # fp8: fwd1 reads the dequantised MXFP8 x, the biases come from the candidates' blobs
            m.set_predicate(self.is_comm_ptr)
            m.mlp_val((self.x_dq if self.fp8 else self.x_bf)[: self.n_val], yv, self.val_correct, self.b_maps,
                      self.dyn_ptr[0], self.dyn_ptr[1], self.n_val, self.in_dim, H,
                      self.spec.by_name["w2"].shape[0], self.world,
                      self.plan_ptr + self.sz["plan_cand_blob_off"] if self.fp8 else 0)
            m.set_predicate(0)
        else:
            self._validate_two_gemms(self.x_bf[: self.n_val], yv, H)
        self._consensus(self.mirror.data_ptr() if (pipe and self.mirror_result) else 0,
                        self.in_seq.data_ptr() if pipe else 0)
        self.launches_per_round = int(m.launch_count() - n0)

    def _validate_two_gemms(self, xv, yv, H):
        m = self.mod
        m.gemm(xv, self.work_shadow, self.h_val, self.n_val, H, self.in_dim, self.world,
               self.in_dim, self.in_dim, 0, 0, False, False, False, G.EPI_GENERIC, 1, H,
               self.n_val * H, 1.0, None, G.ACT_RELU, None, None, 0, None, 1, False, None, 0, 1.0,
               None, None, self.b_maps, None, 0, 0, 0, 0, self.dyn_ptr[0], self.val_bn[0])
        m.gemm(self.h_val, self.work_shadow, None, self.n_val, self.spec.by_name["w2"].shape[0], H,
               self.world, H, H, self.n_val * H, 0, False, False, False, G.EPI_ARGMAX, 1, 0, 0, 1.0,
               None, 0, None, None, 0, None, 1, False, yv, 0, 1.0, None, self.val_correct,
               self.b_maps, None, 0, 0, 0, 0, self.dyn_ptr[1], self.val_bn[1])

    def capture(self):
        """Warm up eagerly (lazy kernel attribute setup), then capture one round."""
        with torch.cuda.stream(self.stream):
            self._enqueue_round()
        self.stream.synchronize()
        self._rounds += 1          # the warm-up is a real round (epoch advanced)
        if not self.cfg.cuda_graph:
            return
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=self.stream):
            self._enqueue_round()
        self.graph = g
        if self.pipelined_input:
            # second graph for run_round_e2e: same round, inputs converted chunk by chunk as
            # their H2D copies land.  Its only new kernel is warmed up once outside the capture
            # (lazy module loading), without running an extra round.
            with torch.cuda.stream(self.stream):
                self.in_seq.fill_(-1)       # the kernel waits for tag *in_seq + 1: 0 = the initial tags
                self.mod.prep_inputs_chunks(self.x_u8, self.x_bf, None, None,
                                            self.cfg.batch_size, self.epoch_steps, 1.0 / 255.0,
                                            self.in_flags, self.in_seq, self.cast_cnt, self.x_ready,
                                            self.in_err, self.x_dq)
                self.in_seq.zero_()         # rounds fed so far (bumped by the consensus kernel)
            self.stream.synchronize()
            gp = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gp, stream=self.stream):
                self._enqueue_round(pipe=True)
            self.graph_pipe = gp
        # raw executable handles for the per-round launch (the captured rounds use no torch RNG, so
        # CUDAGraph.replay()'s generator prologue has nothing to do)
        self._stream_ptr = self.stream.cuda_stream
        if os.environ.get("BFLC_RAW_GRAPH_LAUNCH", "1") != "0":
            for gg in (self.graph, self.graph_pipe):
                try:
                    if gg is not None:
                        self._exec[id(gg)] = int(gg.raw_cuda_graph_exec())
                except Exception:      # older torch: fall back to replay()
                    pass

    @property
    def consensus_captured(self) -> bool:
        return self.graph is not None

    @property
    def graph_train(self):
        """The captured round graph, which holds the DP-SGD noise key (checkpoint adoption checks it)."""
        return self.graph

    @staticmethod
    def _dpsgd_kwargs(cfg: FLConfig, rank: int) -> dict:
        if not cfg.dpsgd_on:
            return {}
        return dict(dpsgd_clip=cfg.dpsgd_clip, dpsgd_noise=cfg.dpsgd_noise, dpsgd_seed=resolve_dpsgd_seed(cfg, rank))

    @property
    def dpsgd_seed(self) -> int:
        return self.trainer.dpsgd_seed if self.dpsgd is not None else 0

    @dpsgd_seed.setter
    def dpsgd_seed(self, seed: int):
        self.dpsgd.seed = seed

    def privacy_spent_local(self) -> Optional[tuple]:
        """(epsilon, delta) of this client's DP-SGD so far, None with DP-SGD off: the generic engine's
        accounting (``GenericFedEngine.privacy_spent_local``) over the same fixed partition batches --
        a record is in at most ceil(opt_total / E) of the opt_total steps, E = batches per epoch."""
        if self.dpsgd is None:
            return None
        from ..utils.checkpoint import plan_counters
        return dpsgd_epsilon(self.cfg, plan_counters(self)[0], self.S // self.cfg.batch_size)

    def run_round(self, pipe: bool = False):
        self._next_round()
        if self._epoch_known is not None:
            self._epoch_known += 1          # every round advances the epoch by exactly one
        g = self.graph_pipe if (pipe and self.graph_pipe is not None) else self.graph
        if g is not None:
            ex = self._exec.get(id(g))
            if ex:      # cudaGraphLaunch straight on the engine stream (no guard, no replay bookkeeping)
                self.mod.graph_launch(ex, self._stream_ptr)
            else:
                with torch.cuda.stream(self.stream):
                    g.replay()
        else:
            with torch.cuda.stream(self.stream):
                self._enqueue_round(pipe=pipe)

    def run_round_e2e(self, host_x: Optional[torch.Tensor] = None,
                      host_y: Optional[torch.Tensor] = None) -> dict:
        """Public per-round call: stage this round's inputs from pinned host memory, run the
        round, read the result (ledger page) back to the host."""
        hx = self.host_x if host_x is None else self._check_host(host_x, self.host_x, "host_x")
        hy = self.host_y if host_y is None else self._check_host(host_y, self.host_y, "host_y")
        if self.pipelined_input:
            # launch the round first, then feed it: labels, chunk 0, tag 0, chunk 1, tag 1, ... on
            # the copy stream; step s of the trainer starts when chunk s has been converted, so
            # the copy of the later chunks hides behind the compute of the earlier steps
            # The copies of round r carry tag r; the device counts fed rounds itself (the consensus
            # kernel bumps in_seq at the end of every pipelined round), so nothing has to be
            # copied in front of the graph.
            self._seq += 1
            self._seq_np[0] = self._seq
            # launch the round, then feed it (issuing chunk 0 ahead of the graph launch waits
            # for the copy before the launch)
            yb = hy.numel() * hy.element_size()
            if self._prefeed:   # labels + chunk 0 travel while the graph launch is in progress
                self.mod.h2d_pipeline(hx.data_ptr(), self._pipe_dst, self._pipe_chunk, 0, 1,
                                      hy.data_ptr(), self._pipe_y, yb, *self._pipe_flags, self._tag_wv)
                self.run_round(pipe=True)
                self.mod.h2d_pipeline(hx.data_ptr(), self._pipe_dst, self._pipe_chunk, 1, self.epoch_steps,
                                      0, 0, 0, *self._pipe_flags, self._tag_wv)
            else:
                self.run_round(pipe=True)
                self.mod.h2d_pipeline(hx.data_ptr(), self._pipe_dst, self._pipe_chunk, 0, self.epoch_steps,
                                      hy.data_ptr(), self._pipe_y, yb, *self._pipe_flags, self._tag_wv)
        else:
            with torch.cuda.stream(self.stream):
                self.x_u8.copy_(hx, non_blocking=True)
                self.y.copy_(hy, non_blocking=True)
            self.run_round()
        if self.pipelined_input and self.mirror_result and self.graph_pipe is not None \
                and self._epoch_known is not None:
            # the kernel wrote the page into pinned memory; every chunk copy was consumed before
            # the trainer's last step, so nothing is in flight once the new epoch is visible
            self._wait_mirror(self._epoch_known)
            return parse_round_state(self._mirror_np, self.world)
        with torch.cuda.stream(self.stream):
            self.out_host.copy_(self.state_bytes, non_blocking=True)
        self.stream.synchronize()
        if self.pipelined_input:
            self._copy_stream.synchronize()
        st = self.read_state(self.out_host)
        self._epoch_known = st["epoch"]
        return st

    def _check_host(self, t: torch.Tensor, like: torch.Tensor, name: str) -> torch.Tensor:
        """A round's host inputs must match the resident pinned ones: the pipeline copies them by raw
        pointer, chunk by chunk, and the plain path copies them non-blocking.  A tensor is checked the
        first time it is passed (is_pinned alone costs microseconds, a few % of a round)."""
        seen = self._host_checked.get(id(t))
        if seen is not None and seen() is t:
            return t
        if not (t.shape == like.shape and t.dtype == like.dtype and t.is_contiguous() and t.is_pinned()):
            raise ValueError(f"run_round_e2e: {name} must be a contiguous pinned {like.dtype} tensor of shape "
                             f"{tuple(like.shape)}, got {t.dtype} {tuple(t.shape)} "
                             f"(contiguous {t.is_contiguous()}, pinned {t.is_pinned()})")
        checked = self._host_checked
        checked[id(t)] = weakref.ref(t, lambda _, k=id(t): checked.pop(k, None))
        return t

    def _wait_mirror(self, want: int):
        m, n, t0 = self._mirror_np, 0, None
        seq = int(self.sz["kMirrorSeqWord"])
        while int(m[seq]) != want:
            n += 1
            if (n & 0x3FFF) == 0:
                now = time.monotonic()
                if t0 is None:
                    t0 = now
                elif now - t0 > 30.0:
                    raise RuntimeError(f"round result never reached the host mirror page (want epoch {want}, "
                                       f"have {int(m[seq])})")

    @property
    def h2d_bytes_per_round(self) -> int:
        tags = 4 * self.epoch_steps if self.pipelined_input else 0   # one 4-byte tag per chunk
        return self.host_x.numel() * self.host_x.element_size() + self.host_y.numel() * 4 + tags

    @property
    def d2h_bytes_per_round(self) -> int:
        if self.pipelined_input and self.mirror_result:
            return int(self.sz["RoundState"]) + 4      # ledger page + epoch word, written by the kernel
        return self.out_host.numel()

    # ------------------------------------------------------------------ host views
    def drain_blocks(self) -> List[str]:
        # Like read_state, this needs nothing but the ledger page, the block ring and the host ledger:
        # it also drains protocol replicas that have no input pipeline (no ``in_err`` word).
        torch.cuda.synchronize()
        in_err = getattr(self, "in_err", None)
        if in_err is not None and int(in_err.item()):
            raise RuntimeError("input pipeline: a chunk's H2D tag never arrived (host stalled > 10 s "
                               "between launching the round and feeding it); the round ran on stale inputs")
        return ProtocolEngine.drain_blocks(self)

    def reset_host_caches(self):
        """Forget the host's copy of the epoch (after a checkpoint restore rewrote the ledger page):
        the next ``run_round_e2e`` re-learns it with one synchronous read."""
        self._epoch_known = None

    @property
    def opt_moments(self) -> tuple:
        """The client optimizer's (m, v) moments, None without Adam."""
        return self.trainer.m, self.trainer.v

    def global_model(self) -> Dict[str, torch.Tensor]:
        return {k: v.clone() for k, v in self.spec.views(self.global_master).items()}

    def evaluate(self, shard: Shard) -> float:
        """Sponsor-style test accuracy of the current global model (M:285-306)."""
        # the global model is written by the round's kernels on the engine stream: wait for them
        torch.cuda.current_stream(self.dev).wait_stream(self.stream)
        x = shard.x.reshape(len(shard), -1).to(self.dev)
        xb = torch.empty(x.shape, device=self.dev, dtype=torch.bfloat16)
        self.mod.prep_inputs(x.contiguous(), xb, None, None, 1.0 / 255.0)
        cnt = self.trainer.accuracy_counts(xb, shard.y.to(self.dev, torch.int32),
                                           shadow=self.global_shadow, master=self.global_master)
        return float(cnt.item()) / len(shard)
