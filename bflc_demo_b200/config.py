"""One runtime configuration object shared by Python and the C++ ledger.

The reference hard-codes its protocol constants twice and keeps them in sync by hand:
C++ ``#define``s (CommitteePrecompiled.h:4-19) and Python module globals
(python-sdk/main.py:52,62,65,68-69,87-88) -- changing the committee size means recompiling
the blockchain node (SURVEY.md 5.6).  Here there is exactly one validated dataclass; the
C++ side receives it through ``to_ledger_config``.
"""
from __future__ import annotations

import dataclasses
import json
import math
import os
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

LR_SCHEDULES = ("constant", "linear", "cosine")   # kernel schedule id = index (bflc_kernels.h)
AGGREGATIONS = ("fedavg", "median", "trimmed_mean")   # rule id = index (consensus_math.hpp AggRule)
SERVER_OPTS = ("none", "momentum", "adam", "yogi")    # optimizer id = index (consensus_math.hpp ServerOpt)
SERVER_LR_DEFAULT = {"momentum": 1.0, "adam": 0.01, "yogi": 0.01}


@dataclass
class FLConfig:
    # ---- protocol (reference names in comments) ----
    clients: int = 20                 # CLIENT_NUM            H:17 / M:52
    committee_size: int = 4           # COMM_COUNT            H:11
    aggregate_count: int = 6          # AGGREGATE_COUNT       H:13
    needed_updates: int = 10          # NEEDED_UPDATE_COUNT   H:15
    learning_rate: float = 0.001      # learning_rate         H:19 / M:88
    max_epoch: int = 1000             # MAX_EPOCH             M:65
    weight_by_score: bool = False     # False = reference (scores filter, n_samples weight)
    # Byzantine-robust aggregation of the selected updates: fedavg (reference) | median |
    # trimmed_mean (coordinate-wise, unweighted; trim updates dropped at each end)
    aggregation: str = "fedavg"
    trim: int = 1
    # server optimizer on the aggregate (pseudo-gradient d = global - aggregate): none (the
    # aggregate is the new model) | momentum (FedAvgM) | adam | yogi (FedAdam / FedYogi, no bias
    # correction).  server_lr 0 = the optimizer's default: 1.0 for momentum, 0.01 for adam / yogi
    server_opt: str = "none"
    server_lr: float = 0.0
    server_beta1: float = 0.9
    server_beta2: float = 0.99
    server_tau: float = 1e-3
    # differentially private aggregation (DP-FedAvg): clip each selected update's model change to L2
    # norm dp_clip (0 = off), add Gaussian noise with multiplier dp_noise to the FedAvg aggregate (0 =
    # clip only), account (epsilon, dp_delta); dp_seed None = rank 0 draws a secret seed at engine
    # construction (a fixed seed lets anyone who holds the config reproduce the noise)
    dp_clip: float = 0.0
    dp_noise: float = 0.0
    dp_delta: float = 1e-5
    dp_seed: Optional[int] = None
    # adaptive clipping of DP-FedAvg (Andrew et al. 2021): dp_clip_quantile 0 = the fixed clip dp_clip;
    # in (0, 1) the clip starts at dp_clip and moves geometrically, at rate dp_clip_lr, toward that
    # quantile of the selected update norms, from a count of unclipped updates noised with
    # dp_count_noise (> dp_noise / 2 with noise, 0 without).  dp_noise stays the total multiplier:
    # epsilon is unchanged, the aggregate's own multiplier is (z^-2 - (2 dp_count_noise)^-2)^-1/2
    dp_clip_quantile: float = 0.0
    dp_clip_lr: float = 0.2
    dp_count_noise: float = 0.0
    # differentially private local training (DP-SGD, ops/dpsgd.py; GenericFedEngine and the host path):
    # clip each example's gradient to L2 norm dpsgd_clip (0 = off) and add Gaussian noise with multiplier
    # dpsgd_noise (0 = clip only) on every local step, with each client's own secret noise key;
    # dpsgd_seed None = every rank draws its key from ``secrets`` (a fixed seed lets anyone who holds the
    # config reproduce, and remove, the noise); the local (epsilon, dp_delta) is privacy_spent_local()
    dpsgd_clip: float = 0.0
    dpsgd_noise: float = 0.0
    dpsgd_seed: Optional[int] = None
    # full-model DP-SGD on bert / gpt (lora_rank 0): every parameter, embeddings and layer norms included,
    # is clipped and noised.  An explicit opt-in: the noise then covers ~10^8 coordinates, not the adapters'
    dpsgd_full_model: bool = False
    # DP-SGD on the convolutional families: lenet5, and resnet18 with resnet_norm "group" (batch norm
    # mixes examples).  An explicit opt-in: convolution sites take per-example patch norms
    dpsgd_conv: bool = False
    # how DP-SGD's local steps pick their examples: "partition" (the fixed batches of engine/base.py step_rows,
    # accounted without amplification) or "poisson" (each record independently with rate batch_size / shard
    # rows, a secret on-device sample in fixed-capacity slots, accounted as the sampled Gaussian mechanism)
    dpsgd_sampling: str = "partition"
    # DP-SGD on the mlp in the persistent trainer (FusedEngine, dtype bf16 or fp8): per-example clipping in
    # the fused chain and the client's noise in the optimizer epilogue.  An explicit opt-in: without it an
    # mlp with dpsgd_clip > 0 runs through GenericFedEngine
    dpsgd_fused: bool = False
    # DP-SGD on packed variable-length bert (--packed): each example's norms over its own tokens, through the
    # segmented per-example kernels.  An explicit opt-in; partition sampling only (a Poisson sample would make
    # each step's token count, and so the captured graph's shapes, depend on the secret sample)
    dpsgd_packed: bool = False
    solo: bool = False                # every client trains and scores (single-GPU runs)
    seed: int = 0
    # ---- model / data ----
    model: str = "mlp"                # softmax | mlp | lenet5 | resnet18 | bert | gpt
    dataset: str = "femnist"          # occupancy | femnist | cifar10 | tokens
    hidden: int = 256                 # MLP hidden width
    resnet_norm: str = "batch"        # resnet18: batch | group (32 groups, per-example statistics)
    batch_size: int = 100             # M:87
    local_epochs: int = 1             # one pass per round (M:141-148)
    samples_per_client: int = 300     # ~ 6107 / 20 in the reference split (A3)
    val_samples: int = 0              # 0 = validate on the whole shard (M:191)
    optimizer: str = "sgd"            # sgd (M:127) | adam (commented alternative, M:126)
    dtype: str = "bf16"               # fp32 | bf16 | fp8
    non_iid_alpha: float = 0.0        # 0 = IID contiguous split (M:43-48); >0 Dirichlet skew
    # ---- fine-tuning optimizer recipe (GenericFedEngine only; ops/optim.py) ----
    # the schedule follows a client's own optimizer-step count; the defaults are the plain optimizer
    weight_decay: float = 0.0         # decoupled (AdamW / torch SGD), never on 1-D parameters
    lr_schedule: str = "constant"     # constant | linear | cosine, after a linear warmup
    warmup_steps: int = 0
    total_steps: int = 0              # end of the linear / cosine decay (must exceed warmup_steps)
    clip_grad_norm: float = 0.0       # > 0: clip the global gradient norm to this (non-finite: skip)
    # ---- FedProx local training (every engine and the host path) ----
    # mu > 0 adds mu/2 ||w - w_g||^2 to the local loss, w_g the global model the round started from:
    # every local step uses g' = fma(mu, w - w_g, g); 0 = plain local training
    prox_mu: float = 0.0
    # ---- LoRA fine-tuning (GenericFedEngine, bert / gpt; models/lora.py) ----
    # rank > 0: the base model is frozen and the update is the low-rank adapters of lora_targets
    lora_rank: int = 0                # 0 = off, else a multiple of 8 in [8, 64]
    lora_alpha: float = 0.0           # adapter scale alpha / rank; 0 = the rank (scale 1)
    lora_targets: str = "q,v"         # comma-separated subset of q,k,v,o,ff1,ff2
    # ---- faults (SURVEY.md 5.3) ----
    byzantine_ranks: List[int] = field(default_factory=list)
    byzantine_scale: float = 5.0
    straggler_ranks: List[int] = field(default_factory=list)   # these clients publish late ...
    straggler_delay_us: int = 0                                # ... by this much (first-K-wins test)
    # ---- engine ----
    backend: str = "auto"             # auto | fused (P2P kernels) | nccl (baseline) | gloo
    two_shot: Optional[bool] = None   # None = by model size
    use_multicast: bool = True
    stage_candidates: bool = True     # committee pulls each candidate's weights once (P2P) vs
                                      # the validation GEMMs TMA-loading peers' HBM directly
    cuda_graph: bool = True
    fused_step: bool = True           # MLP: all local steps of a round in one persistent kernel
    ring_slots: int = 256

    def validate(self) -> "FLConfig":
        c = self
        if c.clients < 1:
            raise ValueError("clients must be >= 1")
        if c.committee_size < 1:
            raise ValueError("committee_size must be >= 1")
        if c.aggregate_count < 1 or c.aggregate_count > c.needed_updates:
            raise ValueError("need 1 <= aggregate_count <= needed_updates")
        if c.solo:
            if c.committee_size > c.clients or c.needed_updates > c.clients:
                raise ValueError("solo: committee_size and needed_updates must be <= clients")
        else:
            # implied (never checked) by the reference: NEEDED <= CLIENT - COMM.  The reference also
            # has COMM <= NEEDED (H:11-15); a committee larger than the trainer set (BASELINE.json
            # config #4: committee 5 of 8) is allowed here: re-election takes every scored
            # trainer and refills from the outgoing committee (consensus_math.hpp step 5).
            if c.needed_updates > c.clients - c.committee_size:
                raise ValueError("needed_updates > clients - committee_size: not enough trainers")
        if not (c.learning_rate > 0):
            raise ValueError("learning_rate must be > 0")
        if not (isinstance(c.local_epochs, int) and c.local_epochs >= 1):
            raise ValueError("local_epochs must be an integer >= 1")
        if c.aggregation not in AGGREGATIONS:
            raise ValueError(f"aggregation must be one of {', '.join(AGGREGATIONS)}")
        if c.aggregation == "trimmed_mean" and not (1 <= c.trim and 2 * c.trim < c.aggregate_count):
            raise ValueError("trimmed_mean needs 1 <= trim and 2 * trim < aggregate_count")
        if c.aggregation != "fedavg" and c.weight_by_score:
            raise ValueError("weight_by_score needs aggregation='fedavg' (median and trimmed mean are unweighted)")
        if c.server_opt not in SERVER_OPTS:
            raise ValueError(f"server_opt must be one of {', '.join(SERVER_OPTS)}")
        if c.server_opt != "none":
            # checked on the fp32 values the kernel and the ledger run with (LedgerConfig::validate)
            with np.errstate(over="ignore"):
                lr, b1, b2, _, _, tau = c.server_opt_constants
            if not (math.isfinite(lr) and lr > 0):
                raise ValueError("server_lr must be finite and > 0 (or 0: the optimizer's default)")
            if not 0 <= b1 < 1:
                raise ValueError("server_beta1 must lie in [0, 1) (in fp32)")
            if c.server_opt in ("adam", "yogi"):
                if not 0 <= b2 < 1:
                    raise ValueError("server_beta2 must lie in [0, 1) (in fp32)")
                if not (math.isfinite(tau) and tau > 0):
                    raise ValueError("server_tau must be finite and > 0")
        # checked on the fp32 values the kernel and the ledger run with (LedgerConfig::validate)
        with np.errstate(over="ignore"):
            clip, noise = c.dp_constants
        if not (math.isfinite(clip) and clip >= 0):
            raise ValueError("dp_clip must be finite and >= 0 (0: off)")
        if not (math.isfinite(noise) and noise >= 0):
            raise ValueError("dp_noise must be finite and >= 0 (0: clip only)")
        if noise > 0 and clip == 0:
            raise ValueError("dp_noise needs dp_clip > 0")
        if noise > 0 and c.aggregation != "fedavg":
            raise ValueError("dp_noise needs aggregation='fedavg' (the L2 sensitivity of a median or a trimmed "
                             "mean is not bounded by dp_clip)")
        q, lr, sb = c.dp_adapt_constants
        if q != 0:
            if not 0 < q < 1:
                raise ValueError("dp_clip_quantile must be 0 (a fixed clip) or lie in (0, 1) (in fp32)")
            if clip == 0:
                raise ValueError("dp_clip_quantile needs dp_clip > 0 (the initial clip)")
            if not (math.isfinite(lr) and lr > 0):
                raise ValueError("dp_clip_lr must be finite and > 0 (in fp32)")
            if noise == 0 and sb != 0:
                raise ValueError("dp_count_noise must be 0 for adaptive clipping without noise (dp_noise 0)")
            if noise > 0 and not (math.isfinite(sb) and 2.0 * float(sb) > float(noise)):
                raise ValueError("dp_count_noise must be finite and > dp_noise / 2: (2 dp_count_noise)^-2 is the "
                                 "count's share of the total dp_noise^-2")
        elif sb != 0:
            raise ValueError("dp_count_noise needs adaptive clipping (dp_clip_quantile > 0)")
        if not 0 < c.dp_delta < 1:
            raise ValueError("dp_delta must lie in (0, 1)")
        if c.dp_seed is not None and not 0 <= c.dp_seed < 1 << 64:
            raise ValueError("dp_seed must be None or an integer in [0, 2^64)")
        with np.errstate(over="ignore"):
            clip, noise = c.dpsgd_constants
        if not (math.isfinite(clip) and clip >= 0):
            raise ValueError("dpsgd_clip must be finite and >= 0 (in fp32; 0: off)")
        if not (math.isfinite(noise) and noise >= 0):
            raise ValueError("dpsgd_noise must be finite and >= 0 (in fp32; 0: clip only)")
        if noise > 0 and clip == 0:
            raise ValueError("dpsgd_noise needs dpsgd_clip > 0")
        if c.dpsgd_seed is not None and not 0 <= c.dpsgd_seed < 1 << 64:
            raise ValueError("dpsgd_seed must be None or an integer in [0, 2^64)")
        if c.dpsgd_sampling not in ("partition", "poisson"):
            raise ValueError("dpsgd_sampling must be partition or poisson")
        if c.dpsgd_sampling == "poisson" and clip == 0:
            raise ValueError("dpsgd_sampling='poisson' needs dpsgd_clip > 0")
        if c.dpsgd_sampling == "poisson" and c.samples_per_client < 2 * c.batch_size:
            raise ValueError("dpsgd_sampling='poisson' samples at rate batch_size / shard rows < 1: it needs "
                             "samples_per_client >= 2 * batch_size")
        if c.dpsgd_full_model:
            if clip == 0:
                raise ValueError("dpsgd_full_model needs dpsgd_clip > 0")
            if c.model not in ("bert", "gpt"):
                raise ValueError(f"dpsgd_full_model applies to bert and gpt, not {c.model}")
            if c.lora_rank > 0:
                raise ValueError("dpsgd_full_model trains the full model: it excludes LoRA (lora_rank > 0)")
        if c.dpsgd_conv:
            if clip == 0:
                raise ValueError("dpsgd_conv needs dpsgd_clip > 0")
            if c.model not in ("lenet5", "resnet18"):
                raise ValueError(f"dpsgd_conv applies to lenet5 and resnet18, not {c.model}")
            if c.model == "resnet18" and c.resnet_norm != "group":
                raise ValueError("dpsgd_conv on resnet18 needs resnet_norm='group': batch norm mixes the examples "
                                 "of a batch, so per-example gradients are not defined")
            if c.dtype == "fp8":
                raise ValueError("dpsgd_conv runs bf16 weight-gradient GEMMs: dtype fp8 is not supported")
        if c.dpsgd_fused:
            if clip == 0:
                raise ValueError("dpsgd_fused needs dpsgd_clip > 0")
            if c.model != "mlp":
                raise ValueError(f"dpsgd_fused applies to the mlp's persistent trainer, not {c.model}")
            if c.dpsgd_sampling != "partition":
                raise ValueError("dpsgd_fused: Poisson sampling needs the generic engine (dpsgd_sampling='partition' "
                                 "only in the persistent trainer)")
            if c.dpsgd_full_model or c.dpsgd_conv or c.lora_rank > 0:
                raise ValueError("dpsgd_fused excludes dpsgd_full_model, dpsgd_conv and LoRA (lora_rank > 0)")
            if not c.fused_step or c.hidden != 256:
                raise ValueError("dpsgd_fused runs in the persistent trainer: it needs fused_step and hidden == 256")
        if c.dpsgd_packed:
            if clip == 0:
                raise ValueError("dpsgd_packed needs dpsgd_clip > 0")
            if c.model != "bert":
                raise ValueError(f"dpsgd_packed applies to packed bert, not {c.model}")
            if c.dpsgd_sampling != "partition":
                raise ValueError("dpsgd_packed needs dpsgd_sampling='partition': a Poisson sample would make each "
                                 "step's token count secret, and a captured step's shapes are fixed")
            if c.dpsgd_conv or c.dpsgd_fused:
                raise ValueError("dpsgd_packed excludes dpsgd_conv and dpsgd_fused")
        if clip > 0:
            if c.model in ("lenet5", "resnet18") and not c.dpsgd_conv:
                raise ValueError(f"DP-SGD (dpsgd_clip > 0) does not cover {c.model}: its convolutions (and "
                                 "ResNet's batch norm, which mixes examples) have no per-example gradient norms here; "
                                 "or opt in with dpsgd_conv")
            if c.model in ("bert", "gpt") and c.lora_rank == 0 and not c.dpsgd_full_model:
                raise ValueError(f"DP-SGD on {c.model} needs LoRA (lora_rank > 0): embeddings and layer norms of "
                                 "the full model have no per-example gradient norms here; or opt in to full-model "
                                 "DP-SGD (dpsgd_full_model)")
            if c.dtype == "fp8" and not c.dpsgd_fused:
                raise ValueError("DP-SGD runs bf16 weight-gradient GEMMs: dtype fp8 is not supported with dpsgd_clip > 0 "
                                 "(or --dpsgd-fused: the persistent trainer's weight gradients are bf16 in both dtypes)")
        if c.resnet_norm not in ("batch", "group"):
            raise ValueError("resnet_norm must be batch or group")
        if c.resnet_norm != "batch" and c.model != "resnet18":
            raise ValueError(f"resnet_norm applies to resnet18 only, not {c.model}")
        if c.optimizer not in ("sgd", "adam"):
            raise ValueError("optimizer must be sgd or adam")
        if c.dtype not in ("fp32", "bf16", "fp8"):
            raise ValueError("dtype must be fp32, bf16 or fp8")
        if not c.weight_decay >= 0:
            raise ValueError("weight_decay must be >= 0")
        if c.lr_schedule not in LR_SCHEDULES:
            raise ValueError(f"lr_schedule must be one of {', '.join(LR_SCHEDULES)}")
        if c.warmup_steps < 0 or c.total_steps < 0:
            raise ValueError("warmup_steps and total_steps must be >= 0")
        if c.lr_schedule != "constant" and c.total_steps <= c.warmup_steps:
            raise ValueError(f"lr_schedule {c.lr_schedule} needs total_steps > warmup_steps")
        if not c.clip_grad_norm >= 0:
            raise ValueError("clip_grad_norm must be >= 0")
        with np.errstate(over="ignore"):
            mu = np.float32(c.prox_mu)
        if not (math.isfinite(mu) and mu >= 0):
            raise ValueError("prox_mu must be finite and >= 0 (in fp32; 0: off)")
        if not (math.isfinite(c.non_iid_alpha) and c.non_iid_alpha >= 0):
            raise ValueError("non_iid_alpha must be finite and >= 0 (0: IID)")
        for r in c.byzantine_ranks:
            if not (0 <= r < c.clients):
                raise ValueError(f"byzantine rank {r} out of range")
        if c.lora_rank != 0:
            from .models.lora import check_rank, parse_targets
            check_rank(c.lora_rank)
            parse_targets(c.lora_targets)
            if c.model not in ("bert", "gpt"):
                raise ValueError(f"LoRA needs model bert or gpt, not {c.model}")
            if c.dtype == "fp8":
                raise ValueError("LoRA runs bf16 GEMMs: dtype fp8 is not supported with lora_rank > 0")
            if not (math.isfinite(c.lora_alpha) and c.lora_alpha >= 0):
                raise ValueError("lora_alpha must be finite and >= 0 (0: the rank)")
        return self

    @property
    def has_optim_recipe(self) -> bool:
        """Any fine-tuning recipe field away from its default (only GenericFedEngine runs them)."""
        return (self.weight_decay != 0 or self.lr_schedule != "constant" or self.warmup_steps != 0
                or self.total_steps != 0 or self.clip_grad_norm != 0)

    @property
    def aggregation_rule(self) -> int:
        """Rule id of the consensus kernel and the ledger (0 FedAvg, 1 median, 2 trimmed mean)."""
        return AGGREGATIONS.index(self.aggregation)

    @property
    def server_opt_id(self) -> int:
        """Server optimizer id of the consensus kernel and the ledger (0 none, 1 momentum, 2 adam, 3 yogi)."""
        return SERVER_OPTS.index(self.server_opt)

    @property
    def server_state_vectors(self) -> int:
        """fp32 [n_params] vectors of server optimizer state: 0 none, 1 momentum (m), 2 adam / yogi (m, v)."""
        return (0, 1, 2, 2)[self.server_opt_id]

    @property
    def server_lr_resolved(self) -> float:
        return self.server_lr or SERVER_LR_DEFAULT.get(self.server_opt, 1.0)

    @property
    def server_opt_constants(self) -> tuple:
        """The six fp32 constants (lr, b1, b2, c1, c2, tau) the kernel, the C++ ledger and the oracle
        run the server step with (c1 = fp32(1 - b1), c2 = fp32(1 - b2), computed in double)."""
        from .protocol.oracle import server_constants
        return server_constants(self.server_lr_resolved, self.server_beta1, self.server_beta2, self.server_tau)

    @property
    def dp_constants(self) -> tuple:
        """(clip, noise multiplier) as the fp32 values the kernel, the C++ ledger and the oracle use."""
        return np.float32(self.dp_clip), np.float32(self.dp_noise)

    @property
    def dp_adapt_constants(self) -> tuple:
        """(quantile, clip rate, count noise) of adaptive clipping as the fp32 values every path uses."""
        with np.errstate(over="ignore"):
            return np.float32(self.dp_clip_quantile), np.float32(self.dp_clip_lr), np.float32(self.dp_count_noise)

    @property
    def dp_adaptive(self) -> bool:
        """Adaptive clipping of DP-FedAvg on (dp_clip_quantile > 0)."""
        return self.dp_mode > 0 and self.dp_adapt_constants[0] != 0

    @property
    def dpsgd_constants(self) -> tuple:
        """(clip, noise multiplier) of DP-SGD as the fp32 values the kernels use."""
        return np.float32(self.dpsgd_clip), np.float32(self.dpsgd_noise)

    @property
    def dpsgd_on(self) -> bool:
        return self.dpsgd_constants[0] > 0

    @property
    def dpsgd_poisson(self) -> bool:
        return self.dpsgd_on and self.dpsgd_sampling == "poisson"

    @property
    def dp_mode(self) -> int:
        """DP mode of the consensus kernel and the ledger: 0 off, 1 clip, 2 clip + noise."""
        clip, noise = self.dp_constants
        return 0 if clip == 0 else 1 if noise == 0 else 2

    @property
    def n_trainers(self) -> int:
        return self.clients if self.solo else self.clients - self.committee_size

    def to_ledger_config(self, model_size: int):
        from ._native import ledger

        L = ledger()
        lc = L.LedgerConfig()
        lc.client_num = self.clients
        lc.comm_count = self.committee_size
        lc.aggregate_count = self.aggregate_count
        lc.needed_update_count = self.needed_updates
        lc.learning_rate = self.learning_rate
        lc.model_size = int(model_size)
        lc.weight_by_score = 1 if self.weight_by_score else 0
        lc.solo = 1 if self.solo else 0
        lc.seed = self.seed
        lc.aggregation = self.aggregation_rule
        lc.trim = self.trim
        lc.server_opt = self.server_opt_id
        lr, b1, b2, _, _, tau = self.server_opt_constants
        lc.server_lr, lc.server_beta1, lc.server_beta2, lc.server_tau = float(lr), float(b1), float(b2), float(tau)
        clip, noise = self.dp_constants
        lc.dp_clip, lc.dp_noise, lc.dp_seed = float(clip), float(noise), int(self.dp_seed or 0)
        q, lr, sb = self.dp_adapt_constants
        lc.dp_clip_quantile, lc.dp_clip_lr, lc.dp_count_noise = float(q), float(lr), float(sb)
        err = lc.validate()
        if err:
            raise ValueError(err)
        return lc

    # ---- construction helpers -------------------------------------------------
    @classmethod
    def reference_default(cls) -> "FLConfig":
        """The reference's own constants: 20 clients, 4 committee, top-6 of 10, lr 1e-3,
        softmax regression 5->2 on UCI Occupancy (H:7-19, M:52-69)."""
        return cls(model="softmax", dataset="occupancy").validate()

    @classmethod
    def reference_scaled(cls, clients: int, **kw) -> "FLConfig":
        """The reference's 20/4/10/6 proportions scaled to another client count."""
        if clients == 20:
            base = dict()
        else:
            comm = max(1, clients // 5)
            trainers = clients - comm
            needed = max(comm, (trainers * 10 + 15) // 16)
            agg = max(1, min(needed, max(comm, (needed * 6 + 9) // 10)))
            base = dict(clients=clients, committee_size=comm, needed_updates=needed,
                        aggregate_count=agg)
        base.update(dict(model="softmax", dataset="occupancy"))
        base.update(kw)
        return cls(**base).validate()

    @classmethod
    def for_world(cls, n: int, committee_size: Optional[int] = None,
                  needed_updates: Optional[int] = None, **kw) -> "FLConfig":
        """The benchmark family of BASELINE.json: n clients, committee 3 at n=8, 2 at n=4,
        1 at n=2, solo at n=1 (``committee_size=5`` gives config #4); by default every trainer's
        update is needed (``needed_updates=k`` < trainers enables first-k-wins admission);
        top-(needed-1) aggregated (at least the committee size when that many are admitted)."""
        if n == 1:
            base = dict(clients=1, committee_size=1, needed_updates=1, aggregate_count=1, solo=True)
        else:
            comm = committee_size or {2: 1, 4: 2, 8: 3}.get(n, max(1, n // 3))
            if not (1 <= comm < n):
                raise ValueError(f"committee_size must be in [1, {n - 1}] for {n} clients")
            trainers = n - comm
            needed = min(needed_updates or trainers, trainers)
            base = dict(clients=n, committee_size=comm, needed_updates=needed,
                        aggregate_count=min(max(comm if comm <= needed else 1, needed - 1, 1), needed))
        base.update(kw)
        return cls(**base).validate()

    @classmethod
    def from_json(cls, text: str) -> "FLConfig":
        return cls(**json.loads(text)).validate()

    @classmethod
    def from_env(cls, prefix: str = "BFLC_", **defaults) -> "FLConfig":
        kw = dict(defaults)
        for f in dataclasses.fields(cls):
            v = os.environ.get(prefix + f.name.upper())
            if v is None:
                continue
            if f.type in ("int", int):
                kw[f.name] = int(v)
            elif f.type in ("float", float):
                kw[f.name] = float(v)
            elif f.type in ("bool", bool):
                kw[f.name] = v.lower() in ("1", "true", "yes")
            elif f.name in ("byzantine_ranks", "straggler_ranks"):
                kw[f.name] = [int(x) for x in v.split(",") if x]
            elif f.name in ("dp_seed", "dpsgd_seed"):
                kw[f.name] = int(v, 0) if v else None
            else:
                kw[f.name] = v
        return cls(**kw).validate()

    def to_json(self) -> str:
        return json.dumps(dataclasses.asdict(self), sort_keys=True)
