"""Model-agnostic federated engine: any ``FlatNet`` (LeNet-5, ResNet-18, BERT-base, GPT, MLP) on the
same device-resident protocol as ``FusedEngine`` -- symmetric-heap upload buffers, epoch-tagged
P2P flags, the consensus/aggregation kernel, the host ledger re-executing every election.

A round is five launches: ``fed_plan_round``, the whole local-training pass as ONE captured
CUDA graph (forward, backward and optimizer of every mini-batch step -- all our kernels, no
host sync), ``fed_upload``, the committee's pull + validation of every candidate as a second
graph, ``fed_consensus_aggregate``.  Which graphs a rank replays is decided from the role
table it read back (104 bytes, pinned, non-blocking) at the end of the previous round -- no
device->host read inside a round.  (``capture()`` is optional: without it the same round runs
eagerly, kernel by kernel.)

Committee validation runs the model *directly on the trainers' HBM*: a candidate's ``Bound`` is a
set of tensor views over the peer-mapped upload buffers, so every GEMM of the forward pass
TMA-loads its weight tiles across NVLink -- the QueryAllUpdates all-gather (reference
C:299-311, M:196-217) never materialises.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.distributed as dist

from ..config import FLConfig
from ..data.packing import PackedTokens
from ..data.synthetic import Shard
from ..models.lora import LoRANet, check_net_matches_config
from ..models.nets import BertBase, Bound, FlatNet
from ..ops.dpsgd import DPSGDStep, PoissonSampler
from ..ops.nn import DropoutRNG
from ..ops.optim import OptimRecipe, RecipeStep
from .base import ROLE_COMM, ROLE_TRAINER, ProtocolEngine, step_rows, vector_ranges


def resolve_dpsgd_seed(cfg: FLConfig, rank: int) -> int:
    """This rank's DP-SGD noise key: 64 bits from ``secrets``, drawn here and never sent anywhere, or,
    with ``cfg.dpsgd_seed`` set (tests), derived from it and the rank -- anyone who holds that seed can
    recompute and remove the noise.  0 without noise and without Poisson sampling (nothing draws from it);
    Poisson sampling keys its secret sample with it even at noise 0."""
    if not cfg.dpsgd_on or (cfg.dpsgd_noise == 0 and not cfg.dpsgd_poisson):
        return 0
    if cfg.dpsgd_seed is None:
        import secrets
        return secrets.randbits(64)
    return (int(cfg.dpsgd_seed) * 0x9E3779B97F4A7C15 + 0xD1B54A32D192ED03 * (rank + 1)) % (1 << 64)


def dpsgd_epsilon(cfg: FLConfig, opt_total: int, batches_per_epoch: int) -> tuple:
    """(epsilon, dp_delta) after ``opt_total`` DP-SGD steps over a fixed partition into
    ``batches_per_epoch`` batches: k = ceil(opt_total / E) steps touch any one record."""
    from ..protocol.privacy import epsilon
    k = -(-int(opt_total) // int(batches_per_epoch))
    z = float(cfg.dpsgd_constants[1])
    if k == 0:
        return 0.0, cfg.dp_delta
    if z == 0:
        return float("inf"), cfg.dp_delta
    return epsilon(z, k, cfg.dp_delta), cfg.dp_delta


def dpsgd_poisson_epsilon(cfg: FLConfig, opt_total: int, q: float, eta: float) -> tuple:
    """(epsilon, delta_total) after ``opt_total`` Poisson-sampled DP-SGD steps at rate q (the sampler's thr /
    2^32): the sampled Gaussian mechanism's RDP, converted at ``dp_delta`` (``privacy.poisson_epsilon``), and
    delta_total = dp_delta + (1 + e^epsilon) opt_total eta for the truncation to the capacity, eta the exact
    overflow probability of one step (the truncated mechanism differs from the untruncated one only on the
    overflow event; DESIGN.md, "DP-SGD")."""
    import math
    from ..protocol.privacy import poisson_epsilon
    z = float(cfg.dpsgd_constants[1])
    eps = poisson_epsilon(q, z, int(opt_total), cfg.dp_delta)
    if not math.isfinite(eps):
        return eps, cfg.dp_delta
    return eps, cfg.dp_delta + (1.0 + math.exp(eps)) * int(opt_total) * eta


class GenericFedEngine(ProtocolEngine):
    def __init__(self, cfg: FLConfig, net: FlatNet, shard: Shard, *, rank: int = 0, world: int = 1,
                 device: int = 0, group=None):
        assert cfg.clients == world and world <= 8
        check_net_matches_config(cfg, net)
        if cfg.dpsgd_on and getattr(net, "packed", False) and not cfg.dpsgd_packed:
            raise ValueError("DP-SGD needs the same rows per example in every layer: packed batches are not supported "
                             "(or opt in with dpsgd_packed)")
        if cfg.dpsgd_packed:
            base = net.base if isinstance(net, LoRANet) else net
            if not (isinstance(base, BertBase) and base.packed):
                raise ValueError("dpsgd_packed needs a packed BertBase (packed=True), bare or under LoRANet")
        epoch_rows = (len(shard) // cfg.batch_size) * cfg.batch_size
        if cfg.dpsgd_poisson and epoch_rows <= cfg.batch_size:
            raise ValueError(f"DP-SGD Poisson sampling needs more shard rows than the batch: this shard gives "
                             f"{epoch_rows} rows per local epoch at batch_size {cfg.batch_size} (use a shard of at "
                             f"least 2 * batch_size rows)")
        self.net = net
        # cfg.dtype "fp8": forward GEMMs of Linear / Conv2d run block-scaled fp8 (ops/mx8.py)
        from ..ops import nn as _nn
        _nn.set_precision("mx8" if cfg.dtype == "fp8" else "bf16")
        super().__init__(cfg, net.spec, shard, net.init_, rank=rank, world=world, device=device, group=group)
        sz, o, hv, P = self.sz, self.layout.offsets, self.heap.view, self.n_params
        # LoRA (models/lora.py): the update is the adapters of a frozen base that each rank holds
        # itself.  Every rank must hold the same base, or the committee would score candidates of
        # different models: compare the base digests over the bootstrap group and refuse a mismatch.
        self.base_digest = None
        if isinstance(net, LoRANet):
            self.base_digest = net.base_digest(self.dev)
            digests = [self.base_digest] * world
            if world > 1:
                dist.all_gather_object(digests, self.base_digest, group=group)
            if len(set(digests)) != 1:
                raise ValueError(f"LoRA base models differ across ranks (sha256 {sorted(set(d[:12] for d in digests))}); "
                                 "every rank must fine-tune the same base")
        self.opt_step_ptr = self.plan_ptr + sz["plan_opt_step_off"]
        # dropout masks (models with dropout): keyed by the plan's optimizer-step word, which
        # fed_plan_round advances every round (and checkpoints restore), plus the step index, with
        # one seed per client
        self.opt_step_word = hv(o["plan"] + sz["plan_opt_step_off"], [1], torch.int32)
        self.dropout_seed = (cfg.seed * 0x9E3779B97F4A7C15 + 0x632BE59BD9B4E019 * (rank + 1)) % (1 << 64)
        self.m = torch.zeros(P, device=self.dev) if cfg.optimizer == "adam" else None
        self.v = torch.zeros(P, device=self.dev) if cfg.optimizer == "adam" else None
        self.bound = net.bind(self.work_master, self.work_shadow, self.grad)
        # fine-tuning recipe (ops/optim.py): its schedule follows the same step word as Adam's bias
        # correction; FedProx runs through the recipe kernel, anchored at this rank's global replica;
        # the default config keeps the plain optimizer step
        self.recipe = OptimRecipe.from_config(cfg)
        self.recipe_step = (None if self.recipe.is_default and cfg.prox_mu == 0 else
                            RecipeStep(self.recipe, net.spec, self.steps, self.dev, anchor=self.global_master,
                                       prox_mu=cfg.prox_mu))
        # DP-SGD (ops/dpsgd.py): per-example clipping and this client's own noise on every local step,
        # keyed by the same step word as dropout; the seed is this rank's secret (never broadcast)
        self.dpsgd_seed = resolve_dpsgd_seed(cfg, rank)
        # Poisson sampling: the steps run at the sampler's capacity, normalised by the expected batch size
        self.poisson = (PoissonSampler(self.S, cfg.batch_size, self.steps, self.dpsgd_seed, self.dev)
                        if cfg.dpsgd_poisson else None)
        slots = self.poisson.cap if self.poisson is not None else cfg.batch_size
        self.dpsgd = (DPSGDStep(net.spec, slots, cfg.dpsgd_clip, cfg.dpsgd_noise, self.dpsgd_seed,
                                self.opt_step_word, self.dev, conv=cfg.dpsgd_conv, norm_batch=cfg.batch_size)
                      if cfg.dpsgd_on else None)
        self._row_loss = None
        self._loss_acc = torch.zeros(1, device=self.dev) if self.poisson is not None else None

        self.x = net.preprocess(shard.x.to(self.dev))
        self.y = shard.y.to(self.dev, torch.int32)
        # big updates take the two-shot FedAvg (reduce a slice, publish it to every replica); small
        # ones the one-shot form.  (The fused engine also switches to two-shot from 8 ranks up; for
        # the generic engine that variant was not measured at 8 GPUs, so it stays opt-in: cfg.two_shot.)
        self.two_shot = cfg.two_shot if cfg.two_shot is not None else (P * 4 > (64 << 20) and world > 1)
        self._peer_bounds = {}
        self._stage = None
        self.n_cand = world if cfg.solo else cfg.n_trainers      # candidates per round (fixed count)
        self.graph_train: Optional[torch.cuda.CUDAGraph] = None
        self.graph_val: Optional[torch.cuda.CUDAGraph] = None
        self.capture_error = ""
        self.stream = torch.cuda.Stream(device=self.dev)
        # role table cache: refreshed from the ledger page at the end of every round
        self._st_host = torch.empty(sz["RoundState"], dtype=torch.uint8).pin_memory()
        self._st_event = torch.cuda.Event()
        self._st = None
        if world > 1:
            dist.barrier(group=group)
        torch.cuda.synchronize()

    @property
    def opt_moments(self) -> tuple:
        """The client optimizer's (m, v) moments, None without Adam."""
        return self.m, self.v

    def reset_host_caches(self):
        """Forget the role table read back at the end of the last round (after a checkpoint restore
        rewrote the ledger page): the next round reads the page synchronously."""
        self._st = None

    # ------------------------------------------------------------------ pieces
    def peer_bound(self, t: int, parity: int) -> Bound:
        key = (t, parity)
        if key not in self._peer_bounds:
            o, P = self.layout.offsets, self.n_params
            master = self.heap.view(o[f"upload_master{parity}"], [P], torch.float32, rank=t)
            shadow = self.heap.view(o[f"upload_shadow{parity}"], [P], torch.bfloat16, rank=t)
            self._peer_bounds[key] = self.net.bind(master, shadow, None)
        return self._peer_bounds[key]

    def local_training(self):
        # DP-SGD: a bit-reproducible step needs activations and input gradients without split-K atomics; the
        # setting holds for this engine's own local steps only, whatever other engines in the process use
        from ..ops import nn as _nn
        prev = _nn.set_deterministic(self.dpsgd is not None)
        try:
            self._local_steps()
        finally:
            _nn.set_deterministic(prev)

    def _local_steps(self):
        if self.poisson is not None:
            self._poisson_steps()
            return
        B = self.cfg.batch_size
        for i in range(self.steps):
            rows = step_rows(i, B, self.S)
            rng = DropoutRNG(self.dropout_seed, self.opt_step_word, i)
            xb = self.x[rows]
            loss = self.net.loss(self.bound, xb, self.y[rows], rng=rng)
            if self.dpsgd is not None:
                # a packed batch's tokens are segmented by example (cfg.dpsgd_packed; the engine refuses it without)
                self.dpsgd.begin(xb if isinstance(xb, PackedTokens) else None)
                try:
                    loss.backward()
                except BaseException:
                    self.dpsgd.abandon()
                    raise
                self.dpsgd.finish(self.grad, i)
            else:
                loss.backward()
            self.loss_sum += loss.detach() * B
            self._optim(i)

    def _optim(self, i: int):
        cfg = self.cfg
        if self.recipe_step is not None:
            self.recipe_step(cfg.optimizer == "adam", self.work_master, self.grad, self.work_shadow,
                             self.m, self.v, cfg.learning_rate, i + 1, self.opt_step_ptr, i)
        else:
            self.mod.optim_step(cfg.optimizer == "adam", self.work_master, self.grad,
                                self.work_shadow, self.m, self.v, cfg.learning_rate, 0.0, 0.9,
                                0.999, 1e-8, i + 1, self.opt_step_ptr, 0, True)

    def _poisson_steps(self):
        """DP-SGD local steps on the secret Poisson sample: one sampler launch for the round, then per step a
        gather of the step's ``cap`` slots (sampled records, then padding), a loss scaled from 1 / cap to 1 / B,
        and the release with the step's count as ``n_valid``.  avg_cost is the mean loss of the sampled examples,
        padding excluded; the upload's n_samples stays the shard's epoch rows, as without sampling."""
        B, ps = self.cfg.batch_size, self.poisson
        ps.sample(self.opt_step_word)
        self._loss_acc.zero_()
        slot = torch.arange(ps.cap, device=self.dev, dtype=torch.int32)
        for i in range(self.steps):
            ids = ps.idx[i]
            xb, yb = self.x.index_select(0, ids), self.y.index_select(0, ids)
            if self._row_loss is None or self._row_loss.numel() != yb.numel():
                self._row_loss = torch.empty(yb.numel(), device=self.dev, dtype=torch.float32)
            rng = DropoutRNG(self.dropout_seed, self.opt_step_word, i)
            loss = self.net.loss(self.bound, xb, yb, rng=rng, row_loss=self._row_loss)
            self.dpsgd.begin()
            try:
                (loss * (ps.cap / B)).backward()
            except BaseException:
                self.dpsgd.abandon()
                raise
            self.dpsgd.finish(self.grad, i, n_valid=ps.count[i:i + 1])
            per_ex = self._row_loss.view(ps.cap, -1).mean(1)
            self._loss_acc += torch.where(slot < ps.count[i], per_ex, 0.0).sum(0, keepdim=True)
            self._optim(i)
        # fed_upload divides loss_sum by the nominal steps * B
        total = ps.count.sum(0, keepdim=True).clamp_(min=1).float()
        self.loss_sum.copy_(self._loss_acc * float(self.steps * B) / total)

    def privacy_spent_local(self) -> Optional[tuple]:
        """(epsilon, delta) of this client's DP-SGD so far against add/remove-one-record adjacency, None
        with DP-SGD off.  Each local step is a Gaussian mechanism with sensitivity C and noise z C; the
        steps read the fixed batches of ``step_rows``, so a record is in at most k = ceil(opt_total / E)
        of the opt_total steps, E = batches per epoch, and k steps compose to sqrt(k) / z GDP
        (``privacy.epsilon``).  No amplification by subsampling is claimed for these partition batches; Poisson
        sampling returns ``dpsgd_poisson_epsilon``'s (epsilon, delta_total) instead.  Reads the plan page
        (a device->host copy).  Clipping without noise (z = 0) gives no guarantee: epsilon is inf."""
        if self.dpsgd is None:
            return None
        from ..utils.checkpoint import plan_counters
        if self.poisson is not None:   # (dpsgd_sampling "poisson": the amplified accounting instead)
            return dpsgd_poisson_epsilon(self.cfg, plan_counters(self)[0], self.poisson.q, self.poisson.eta)
        return dpsgd_epsilon(self.cfg, plan_counters(self)[0], self.S // self.cfg.batch_size)

    @property
    def grad_norms(self) -> Optional[torch.Tensor]:
        """Pre-clip global gradient norm of each local step of the last round (clipping on)."""
        r = self.recipe_step
        return r.norms if r is not None and self.recipe.clip_grad_norm > 0 else None

    @property
    def skipped_steps(self) -> Optional[torch.Tensor]:
        """int32 [1]: local steps skipped for a non-finite gradient norm (clipping on)."""
        r = self.recipe_step
        return r.skipped if r is not None and self.recipe.clip_grad_norm > 0 else None

    def _vector_ranges(self) -> torch.Tensor:
        return vector_ranges(self.net.spec).to(self.dev)

    def _ensure_stage(self):
        if self._stage is None:
            P = self.n_params
            self._ranges = self._vector_ranges()
            self._stage = (torch.empty(self.world, P, device=self.dev, dtype=torch.bfloat16),
                           torch.empty(self.world, P, device=self.dev, dtype=torch.float32))
            self._stage_bounds = [self.net.bind(self._stage[1][z], self._stage[0][z], None)
                                  for z in range(self.world)]

    def validate_staged(self):
        """Committee: one P2P pass per candidate (bf16 weights + fp32 master) into local staging,
        started per candidate as soon as its trainer's flag is up (the kernel resolves the
        candidate -> trainer mapping from the ledger page), then the forward pass of every
        candidate slot out of local HBM.  No host-side knowledge of who the trainers are: the
        sequence is identical every round and therefore capturable."""
        xv, yv = self.x[: self.n_val], self.y[: self.n_val]
        self._ensure_stage()
        self.mod.fed_pull_candidates(self.fed, self._stage[0], self._stage[1],
                                     self._ranges if self._ranges.numel() else None)
        for z in range(self.n_cand):
            cnt = self.net.correct(self._stage_bounds[z], xv, yv)
            self.val_correct[z:z + 1].copy_(cnt)

    def validate(self, trainers: List[int], parity: int):
        xv, yv = self.x[: self.n_val], self.y[: self.n_val]
        if self.staged:
            self.validate_staged()
            return
        else:
            # direct: every GEMM of the forward pass TMA-loads its weight tiles from the peer
            self.mod.fed_wait_trained(self.fed)
            bounds = [self.peer_bound(t, parity) for t in trainers]
        for z, b in enumerate(bounds):
            cnt = self.net.correct(b, xv, yv)
            self.val_correct[z:z + 1].copy_(cnt)

    # ------------------------------------------------------------------ graphs
    def capture(self):
        """Warm up with one real (eager) round -- lazy kernel attribute setup, autograd graph
        buffers -- then capture the local-training pass and the staged validation pass.  Collective:
        every rank calls it.  Falls back to eager rounds if a capture fails (``capture_error``)."""
        self.run_round()
        torch.cuda.synchronize()
        if self.world > 1:
            dist.barrier(group=self.group)
        if not self.cfg.cuda_graph:
            return
        # A rank that was committee in the warm-up round has never run the training body (and a
        # trainer never the validation forward): do both once, eagerly, on saved-and-restored
        # state, so that no first-use initialisation (lazy module loading, per-thread context
        # binding of autograd's worker, buffer caches) happens inside a capture.
        with torch.cuda.stream(self.stream):
            state = [t for t in (self.work_master, self.work_shadow, self.grad, self.m, self.v, self.grad_norms,
                                 self.skipped_steps, self.dpsgd and self.dpsgd.dropped,
                                 self.poisson and self.poisson.overflow) if t is not None]
            keep = [t.clone() for t in state]
            plan = self.plan_bytes.clone()
            self.local_training()
            self.net.correct(self.bound, self.x[: self.n_val], self.y[: self.n_val])
            for t, k in zip(state, keep):
                t.copy_(k)
            self.plan_bytes.copy_(plan)
        torch.cuda.synchronize()
        del keep, plan
        try:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=self.stream):
                self.local_training()
            self.graph_train = g
            if self.staged:      # (direct validation reads parity/trainer-dependent peer views: eager)
                gv = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gv, stream=self.stream):
                    self.validate_staged()
                self.graph_val = gv
        except Exception as e:  # noqa: BLE001
            self.graph_train = self.graph_val = None
            self.capture_error = repr(e)
        torch.cuda.synchronize()
        if self.world > 1:
            dist.barrier(group=self.group)

    def _roles(self) -> dict:
        """Role table of the round about to start: read back at the end of the previous round."""
        if self._st is None:
            return self.read_state()
        self._st_event.synchronize()
        return self.read_state(self._st_host)

    # ------------------------------------------------------------------ one round
    def run_round(self) -> dict:
        m, cfg = self.mod, self.cfg
        self._next_round()
        st = self._roles()
        role = st["roles"][self.rank]
        trainers = [r for r in range(self.world) if st["roles"][r] & ROLE_TRAINER]
        with torch.cuda.stream(self.stream):
            m.fed_plan_round(self.fed, [], self.steps, False)
            if role & ROLE_TRAINER:
                if self.graph_train is not None:
                    self.graph_train.replay()
                else:
                    self.local_training()
            m.fed_upload(self.fed, self.S, self.steps * cfg.batch_size, self.byz, cfg.byzantine_scale,
                         self.straggle_us)
            if role & ROLE_COMM:
                if self.graph_val is not None:
                    self.graph_val.replay()
                else:
                    self.validate(trainers, st["epoch"] & 1)
            self._consensus()
            # next round's role table: non-blocking readback of the ledger page
            self._st_host.copy_(self.state_bytes, non_blocking=True)
            self._st_event.record(self.stream)
            self._st = True
        torch.cuda.current_stream().wait_stream(self.stream)
        return st

    def evaluate(self, shard: Shard) -> float:
        x = self.net.preprocess(shard.x.to(self.dev))
        y = shard.y.to(self.dev, torch.int32)
        b = self.net.bind(self.global_master, self.global_shadow, None)
        return float(self.net.correct(b, x, y).item()) / y.numel()     # per target (next-token: per position)
