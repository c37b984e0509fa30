"""Command-line runner for the GPU engines (the counterpart of ``python main.py`` in the
reference, python-sdk/main.py:343-358, for one NVSwitch box):

    python -m bflc_demo_b200.run --model mlp --rounds 20                       # 1 GPU, solo
    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 \\
        -m bflc_demo_b200.run --model resnet18 --rounds 5 --byzantine 7       # config #4

BASELINE.json configs: ``--model mlp`` (#2), ``lenet5`` (#3, non-IID CIFAR shards), ``resnet18``
(#4, use --byzantine), ``bert`` (#5, seq_len 128; ``--seq-len`` up to 512 and ``--min-seq-len``
for right-padded variable-length batches, ``--packed`` to run every layer on the real tokens only,
``--dropout P`` for training dropout), ``gpt`` (next-token prediction on a topic-mixture bigram corpus
with a causal decoder of ``--gpt-layers`` layers; ``--seq-len``, ``--dropout``, and ``--non-iid-alpha``
for the clients' topic skew).  ``--weight-decay``, ``--lr-schedule``, ``--warmup-steps``,
``--total-steps`` and ``--clip-grad-norm`` select the fine-tuning optimizer recipe (generic engine
only; ops/optim.py).  ``--prox-mu`` turns on FedProx local training (every model, both engines) and
``--non-iid-alpha`` sets the Dirichlet label skew of the clients' shards.  ``--lora-rank`` (bert, gpt)
freezes the base model (``--lora-base``: a full run's ``--checkpoint``) and trains low-rank adapters
(``--lora-alpha``, ``--lora-targets``), which are then the whole update.  ``--dpsgd-clip`` /
``--dpsgd-noise`` / ``--dpsgd-seed`` (/ ``--dpsgd-sampling poisson``) turn on DP-SGD local training (generic MLP, LoRA BERT / GPT, and
full BERT / GPT with ``--dpsgd-full-model``, LeNet-5 and the GroupNorm ResNet-18 with ``--dpsgd-conv``,
``--packed`` BERT with ``--dpsgd-packed``) and
print each round's local epsilon.  Rank 0 doubles as
the sponsor: after every round it evaluates the global model on a held-out test shard and prints the
reference's two log lines (``the E epoch , global loss : L`` / ``Epoch: 00E, test_acc: A``).
"""
from __future__ import annotations

import argparse
import json
import os
import time

import torch
import torch.distributed as dist

from .config import AGGREGATIONS, LR_SCHEDULES, SERVER_OPTS, FLConfig
from .data.synthetic import cifar_like, femnist_like, lm_corpus_like, tokens_like
from .utils.metrics import RunLog
from .utils.tracing import PhaseTimer


def check_seq_args(ap: argparse.ArgumentParser, seq_len: int, min_seq_len):
    """--seq-len must suit the fused attention kernels and BERT's 512 positions: a multiple of 64
    in [64, 512].  --min-seq-len defaults to --seq-len and must lie in [1, --seq-len]."""
    if seq_len % 64 != 0 or not 64 <= seq_len <= 512:
        ap.error(f"--seq-len {seq_len}: must be a multiple of 64 in [64, 512]")
    min_seq = seq_len if min_seq_len is None else min_seq_len
    if not 1 <= min_seq <= seq_len:
        ap.error(f"--min-seq-len {min_seq}: must lie in [1, --seq-len]")
    return seq_len, min_seq


def add_recipe_args(ap: argparse.ArgumentParser):
    """Flags of the fine-tuning optimizer recipe (GenericFedEngine; ops/optim.py)."""
    ap.add_argument("--weight-decay", type=float, default=0.0,
                    help="decoupled weight decay (AdamW / torch SGD); biases, norm parameters and running "
                         "statistics are never decayed (default 0)")
    ap.add_argument("--lr-schedule", default="constant", choices=list(LR_SCHEDULES),
                    help="learning-rate factor after the warmup, over a client's own optimizer steps")
    ap.add_argument("--warmup-steps", type=int, default=0, help="linear lr warmup from 0 (default 0)")
    ap.add_argument("--total-steps", type=int, default=None,
                    help="linear / cosine: step at which the decay ends (default: rounds x local steps per "
                         "round, the most optimizer steps one client can take in the run)")
    ap.add_argument("--clip-grad-norm", type=float, default=0.0,
                    help="> 0: clip the global gradient norm to this value; a step with a non-finite norm is "
                         "skipped (default 0: no clipping)")


def add_local_args(ap: argparse.ArgumentParser):
    """Flags of the clients' local training: FedProx and the label skew of their shards."""
    ap.add_argument("--prox-mu", type=float, default=0.0,
                    help="FedProx: add mu/2 ||w - w_global||^2 to the local loss, w_global the model the round "
                         "started from (default 0: plain local training)")
    ap.add_argument("--non-iid-alpha", type=float, default=None,
                    help="Dirichlet(alpha) label skew of every client's shard, 0 = IID (default: the model's "
                         "own split)")


def local_fields(ap: argparse.ArgumentParser, a) -> dict:
    """FLConfig fields of the local-training flags, validated (a bad value exits with code 2)."""
    kw = dict(prox_mu=a.prox_mu)
    if a.non_iid_alpha is not None:
        kw["non_iid_alpha"] = a.non_iid_alpha
    try:
        FLConfig(**kw).validate()
    except ValueError as e:
        ap.error(f"local training: {e}")
    return kw


def add_lora_args(ap: argparse.ArgumentParser):
    """Flags of LoRA fine-tuning (bert, gpt; GenericFedEngine; models/lora.py)."""
    ap.add_argument("--lora-rank", type=int, default=0,
                    help="bert, gpt: freeze the base model and train rank-r adapters (a multiple of 8 in "
                         "[8, 64]); the update every round uploads is the adapters only (default 0: off)")
    ap.add_argument("--lora-alpha", type=float, default=0.0,
                    help="adapter scale alpha / rank (default 0: alpha = rank, scale 1)")
    ap.add_argument("--lora-targets", default="q,v",
                    help="comma-separated projections that get adapters: q,k,v,o,ff1,ff2 (default q,v)")
    ap.add_argument("--lora-base", default="",
                    help="the frozen base: a --checkpoint file of a full run of the same model and shape, "
                         "read by every rank (default: the model's seeded genesis)")


def lora_fields(ap: argparse.ArgumentParser, a) -> dict:
    """FLConfig fields of the LoRA flags, validated (a bad value or combination exits with code 2)."""
    if a.lora_rank == 0:
        if a.lora_alpha or a.lora_targets != "q,v" or a.lora_base:
            ap.error("--lora-alpha / --lora-targets / --lora-base need --lora-rank")
        return {}
    if a.model not in ("bert", "gpt"):
        ap.error(f"--lora-rank applies to --model bert and gpt only (not {a.model})")
    kw = dict(lora_rank=a.lora_rank, lora_alpha=a.lora_alpha, lora_targets=a.lora_targets)
    try:
        FLConfig(model=a.model, **kw).validate()
    except ValueError as e:
        ap.error(f"LoRA: {e}")
    if a.lora_base and not (os.path.exists(a.lora_base) or os.path.exists(a.lora_base + ".rank0")):
        ap.error(f"--lora-base {a.lora_base}: no such checkpoint")
    return kw


def add_aggregation_args(ap: argparse.ArgumentParser):
    """Flags of the aggregation rule applied to the committee's selected updates."""
    ap.add_argument("--aggregation", default="fedavg", choices=list(AGGREGATIONS),
                    help="fedavg (sample-weighted mean, default), or the Byzantine-robust coordinate-wise "
                         "median / trimmed_mean of the selected updates")
    ap.add_argument("--trim", type=int, default=1,
                    help="trimmed_mean: updates dropped at each end of every coordinate, "
                         "1 <= trim and 2 * trim < aggregate_count (default 1)")


def add_server_opt_args(ap: argparse.ArgumentParser):
    """Flags of the server optimizer applied to the aggregate of the selected updates."""
    ap.add_argument("--server-opt", default="none", choices=list(SERVER_OPTS),
                    help="none (the aggregate is the new global model, default), or a server optimizer on the "
                         "pseudo-gradient global - aggregate: momentum (FedAvgM), adam (FedAdam), yogi (FedYogi)")
    ap.add_argument("--server-lr", type=float, default=0.0,
                    help="server learning rate (default 0: 1.0 for momentum, 0.01 for adam / yogi)")
    ap.add_argument("--server-beta1", type=float, default=0.9, help="first-moment decay in [0, 1) (default 0.9)")
    ap.add_argument("--server-beta2", type=float, default=0.99,
                    help="adam / yogi: second-moment decay in [0, 1) (default 0.99)")
    ap.add_argument("--server-tau", type=float, default=1e-3,
                    help="adam / yogi: adaptivity tau > 0 added to sqrt(v) (default 1e-3)")


def server_opt_fields(ap: argparse.ArgumentParser, a) -> dict:
    """FLConfig fields of the server optimizer flags, validated (a bad value exits with code 2)."""
    kw = dict(server_opt=a.server_opt, server_lr=a.server_lr, server_beta1=a.server_beta1,
              server_beta2=a.server_beta2, server_tau=a.server_tau)
    try:
        FLConfig(**kw).validate()
    except ValueError as e:
        ap.error(f"server optimizer: {e}")
    return kw


def add_dp_args(ap: argparse.ArgumentParser):
    """Flags of differentially private aggregation (DP-FedAvg) of the selected updates."""
    ap.add_argument("--dp-clip", type=float, default=0.0,
                    help="clip each selected update's model change to this L2 norm (default 0: off)")
    ap.add_argument("--dp-noise", type=float, default=0.0,
                    help="Gaussian noise multiplier z on the FedAvg aggregate, sigma = z * clip * max weight "
                         "(default 0: clip only)")
    ap.add_argument("--dp-delta", type=float, default=1e-5, help="delta of the reported (epsilon, delta) (default 1e-5)")
    ap.add_argument("--dp-seed", type=lambda s: int(s, 0), default=None,
                    help="noise seed (default: 64 secret bits drawn by rank 0; a fixed seed lets anyone who "
                         "knows it reproduce, and remove, the noise)")
    ap.add_argument("--dp-clip-quantile", type=float, default=0.0,
                    help="adaptive clipping: move the clip each round toward this quantile of the selected update "
                         "norms, starting from --dp-clip (default 0: a fixed clip)")
    ap.add_argument("--dp-clip-lr", type=float, default=0.2,
                    help="adaptive clipping: geometric rate of the clip update (default 0.2)")
    ap.add_argument("--dp-count-noise", type=float, default=0.0,
                    help="adaptive clipping: noise on the count of unclipped updates, > --dp-noise / 2 with "
                         "noise, 0 without; --dp-noise stays the total multiplier (default 0)")


def dp_fields(ap: argparse.ArgumentParser, a) -> dict:
    """FLConfig fields of the DP flags, validated against --aggregation (a bad value exits with code 2)."""
    kw = dict(dp_clip=a.dp_clip, dp_noise=a.dp_noise, dp_delta=a.dp_delta, dp_seed=a.dp_seed,
              dp_clip_quantile=a.dp_clip_quantile, dp_clip_lr=a.dp_clip_lr, dp_count_noise=a.dp_count_noise)
    try:
        FLConfig(aggregation=a.aggregation, **kw).validate()
    except ValueError as e:
        ap.error(f"differential privacy: {e}")
    return kw


def add_dpsgd_args(ap: argparse.ArgumentParser):
    """Flags of differentially private local training (DP-SGD, ops/dpsgd.py; generic engine)."""
    ap.add_argument("--dpsgd-clip", type=float, default=0.0,
                    help="clip each example's gradient to this L2 norm on every local step (default 0: off)")
    ap.add_argument("--dpsgd-noise", type=float, default=0.0,
                    help="Gaussian noise multiplier z of each local step, std z * clip / batch per coordinate "
                         "(default 0: clip only)")
    ap.add_argument("--dpsgd-seed", type=lambda s: int(s, 0), default=None,
                    help="derive every client's noise key from this seed (default: 64 secret bits per client; a "
                         "fixed seed lets anyone who knows it reproduce, and remove, the noise)")
    ap.add_argument("--dpsgd-full-model", action="store_true",
                    help="DP-SGD on every parameter of a full bert / gpt run (no --lora-rank): embeddings, layer "
                         "norms and the tied head included")
    ap.add_argument("--dpsgd-conv", action="store_true",
                    help="DP-SGD on lenet5, or on resnet18 with --resnet-norm group: per-example norms of every "
                         "convolution and group norm")
    ap.add_argument("--dpsgd-fused", action="store_true",
                    help="DP-SGD on the mlp in the persistent trainer (FusedEngine, bf16 or fp8) instead of the "
                         "generic engine")
    ap.add_argument("--dpsgd-packed", action="store_true",
                    help="DP-SGD on --packed bert (LoRA or --dpsgd-full-model): each example's gradient norm over "
                         "its own tokens")
    ap.add_argument("--dpsgd-sampling", default="partition", choices=["partition", "poisson"],
                    help="how local steps pick examples: partition (fixed batches, default) or poisson (each record "
                         "with probability batch / shard size, a secret sample, amplified accounting)")


def dpsgd_fields(ap: argparse.ArgumentParser, a) -> dict:
    """FLConfig fields of the DP-SGD flags, refused where DP-SGD does not run (exit code 2)."""
    kw = dict(dpsgd_clip=a.dpsgd_clip, dpsgd_noise=a.dpsgd_noise, dpsgd_seed=a.dpsgd_seed,
              dpsgd_full_model=a.dpsgd_full_model, dpsgd_conv=a.dpsgd_conv, dpsgd_sampling=a.dpsgd_sampling,
              dpsgd_fused=a.dpsgd_fused, dpsgd_packed=a.dpsgd_packed)
    if a.dpsgd_clip == 0 and (a.dpsgd_noise or a.dpsgd_seed is not None):
        ap.error("--dpsgd-noise / --dpsgd-seed need --dpsgd-clip")
    if a.dpsgd_clip == 0 and a.dpsgd_full_model:
        ap.error("--dpsgd-full-model needs --dpsgd-clip")
    if a.dpsgd_clip == 0 and a.dpsgd_conv:
        ap.error("--dpsgd-conv needs --dpsgd-clip")
    if a.dpsgd_clip == 0 and a.dpsgd_sampling != "partition":
        ap.error("--dpsgd-sampling poisson needs --dpsgd-clip")
    if a.dpsgd_clip == 0 and a.dpsgd_fused:
        ap.error("--dpsgd-fused needs --dpsgd-clip")
    if a.dpsgd_packed and a.dpsgd_clip == 0:
        ap.error("--dpsgd-packed needs --dpsgd-clip")
    if a.dpsgd_packed and not a.packed:
        ap.error("--dpsgd-packed needs --packed")
    if a.dpsgd_fused:
        if a.model != "mlp":
            ap.error(f"--dpsgd-fused applies to --model mlp, not {a.model}")
        if a.generic:
            ap.error("--dpsgd-fused runs the persistent trainer: it excludes --generic")
        if a.dpsgd_sampling != "partition":
            ap.error("--dpsgd-fused: Poisson sampling needs the generic engine (drop --dpsgd-fused)")
    if a.dpsgd_clip:
        if a.model == "mlp" and not a.generic and not a.dpsgd_fused:
            ap.error("--dpsgd-clip needs the generic engine: the fused MLP trainer has no per-example clipping "
                     "(add --generic, or --dpsgd-fused)")
        if a.packed and not a.dpsgd_packed:
            ap.error("--dpsgd-clip does not support --packed (rows per example vary there; or --dpsgd-packed)")
    try:
        norm = dict(resnet_norm=a.resnet_norm) if a.model == "resnet18" and a.resnet_norm else {}
        FLConfig(model=a.model, dtype=a.dtype, lora_rank=a.lora_rank, **norm, **kw).validate()
    except ValueError as e:
        ap.error(f"DP-SGD: {e}")
    return kw


def recipe_fields(ap: argparse.ArgumentParser, a, max_steps: int) -> dict:
    """FLConfig fields of the recipe flags, validated (a bad value exits with code 2).  ``max_steps``
    is the default --total-steps of a decaying schedule."""
    total = a.total_steps
    if total is None:
        total = max_steps if a.lr_schedule != "constant" else 0
    kw = dict(weight_decay=a.weight_decay, lr_schedule=a.lr_schedule, warmup_steps=a.warmup_steps,
              total_steps=total, clip_grad_norm=a.clip_grad_norm)
    try:
        FLConfig(**kw).validate()
    except ValueError as e:
        ap.error(f"optimizer recipe: {e}")
    return kw


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="mlp", choices=["mlp", "lenet5", "resnet18", "bert", "gpt"])
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--samples", type=int, default=0, help="samples per client (0 = model default)")
    ap.add_argument("--batch", type=int, default=0)
    ap.add_argument("--lr", type=float, default=0.0)
    ap.add_argument("--optimizer", default=None, choices=["sgd", "adam"],
                    help="client optimizer (default: adam for gpt, sgd otherwise)")
    ap.add_argument("--byzantine", type=int, nargs="*", default=[])
    ap.add_argument("--bert-layers", type=int, default=12)
    ap.add_argument("--gpt-layers", type=int, default=12)
    ap.add_argument("--checkpoint", default="")
    ap.add_argument("--resume", default="")
    ap.add_argument("--no-stage", action="store_true", help="validate straight out of peers' HBM")
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "fp8"],
                    help="fp8: block-scaled (MXFP8) forward GEMMs (the MLP keeps the fused persistent trainer)")
    ap.add_argument("--generic", action="store_true", help="run the MLP through GenericFedEngine")
    ap.add_argument("--seq-len", type=int, default=128, help="bert, gpt: token positions per sample")
    ap.add_argument("--min-seq-len", type=int, default=None,
                    help="bert: shortest sample (default --seq-len); shorter samples are right-padded "
                         "with token 0 and attention masks the padding")
    ap.add_argument("--packed", action="store_true",
                    help="bert: pack each mini-batch's real tokens (token 0 is padding) so that every layer "
                         "runs on them only, and attention on cu_seqlens")
    ap.add_argument("--dropout", type=float, default=0.0,
                    help="bert, gpt: dropout probability in [0, 1) at the embeddings, attention probabilities, "
                         "attention and FFN outputs (and bert's pooled vector; training only; default 0)")
    ap.add_argument("--resnet-norm", default=None, choices=["batch", "group"],
                    help="resnet18: batch norm (default) or group norm (32 groups, per-example statistics, no "
                         "running statistics in the model)")
    add_recipe_args(ap)
    add_aggregation_args(ap)
    add_server_opt_args(ap)
    add_dp_args(ap)
    add_local_args(ap)
    add_lora_args(ap)
    add_dpsgd_args(ap)
    a = ap.parse_args(argv)
    server = server_opt_fields(ap, a)
    dp = dp_fields(ap, a)
    local = local_fields(ap, a)
    lora = lora_fields(ap, a)
    dpsgd = dpsgd_fields(ap, a)
    if lora and a.dtype == "fp8":
        ap.error("--lora-rank runs bf16 GEMMs: --dtype fp8 is not supported with LoRA")
    seq_len, min_seq = check_seq_args(ap, a.seq_len, a.min_seq_len)
    if a.packed and a.model != "bert":
        ap.error("--packed applies to --model bert only")
    if a.min_seq_len is not None and a.model == "gpt":
        ap.error("--min-seq-len does not apply to --model gpt (causal attention runs on full-length samples)")
    if a.non_iid_alpha is not None and a.model == "bert":
        ap.error("--non-iid-alpha applies to --model mlp, lenet5, resnet18 and gpt (the token shards have no label skew)")
    if a.dropout and a.model not in ("bert", "gpt"):
        ap.error("--dropout applies to --model bert and gpt only")
    if not 0.0 <= a.dropout < 1.0:
        ap.error(f"--dropout {a.dropout}: must lie in [0, 1)")
    if a.resnet_norm is not None and a.model != "resnet18":
        ap.error("--resnet-norm applies to --model resnet18 only")
    resnet_norm = a.resnet_norm or "batch"
    defaults = dict(mlp=(4096, 512, 0.05), lenet5=(2048, 128, 0.05), resnet18=(512, 64, 0.02),
                    bert=(64, 16, 0.002), gpt=(2048, 16, 1e-3))[a.model]
    optimizer = a.optimizer or ("adam" if a.model == "gpt" else "sgd")
    S, B, LR = a.samples or defaults[0], a.batch or defaults[1], a.lr or defaults[2]
    recipe = recipe_fields(ap, a, a.rounds * (S // B))      # one local epoch per round
    if a.model == "mlp" and not a.generic and FLConfig(**recipe).has_optim_recipe:
        ap.error("--weight-decay / --lr-schedule / --warmup-steps / --total-steps / --clip-grad-norm need "
                 "the generic engine: the fused MLP trainer has no such optimizer (add --generic)")

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    lr_ = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(lr_)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", lr_))

    try:
        cfg = FLConfig.for_world(world, model=a.model, batch_size=B, samples_per_client=S,
                                 learning_rate=LR, optimizer=optimizer, byzantine_ranks=a.byzantine,
                                 stage_candidates=not a.no_stage, ring_slots=1024, dtype=a.dtype,
                                 aggregation=a.aggregation, trim=a.trim, resnet_norm=resnet_norm, **server, **dp,
                                 **recipe, **local, **lora, **dpsgd)
    except ValueError as e:
        ap.error(str(e))
    if a.model == "mlp":
        shard = femnist_like(world, S, seed=7, only=rank, alpha=cfg.non_iid_alpha)[0]
        test = femnist_like(1, 2048, seed=7, only=0)[0]
    elif a.model in ("lenet5", "resnet18"):
        alpha = 0.5 if a.non_iid_alpha is None else a.non_iid_alpha
        shard = cifar_like(world, S, seed=7, alpha=alpha)[rank]
        test = cifar_like(1, 1024, seed=7, alpha=0.0)[0]
    elif a.model == "gpt":
        alpha = 0.0 if a.non_iid_alpha is None else a.non_iid_alpha
        shard = lm_corpus_like(world, S, seed=7, seq_len=seq_len, alpha=alpha, only=rank)[0]
        test = lm_corpus_like(1, 64, seed=7, seq_len=seq_len, only=0)[0]
    else:
        # packed: token 0 marks padding, so real tokens must avoid it even at full length
        padded = min_seq < seq_len or a.packed
        kw = dict(seq_len=seq_len, min_len=min_seq if padded else None)
        shard = tokens_like(world, S, seed=7, **kw)[rank]
        test = tokens_like(1, 128, seed=8, **kw)[0]

    if a.model == "mlp" and not a.generic:
        from .engine.fused import FusedEngine
        eng = FusedEngine(cfg, shard, rank=rank, world=world, device=lr_)
        eng.capture()
    else:
        from .engine.generic import GenericFedEngine
        from .models.nets import build_model
        pad_id = 0 if (a.model == "bert" and (min_seq < seq_len or a.packed)) else None
        net = build_model(a.model, shard.n_classes, layers=a.gpt_layers if a.model == "gpt" else a.bert_layers,
                          pad_id=pad_id, packed=a.packed, dropout=a.dropout, norm=cfg.resnet_norm)
        if cfg.lora_rank:
            from .models.lora import lora_net_from_config
            try:
                net = lora_net_from_config(cfg, net, a.lora_base or None)
            except ValueError as e:
                ap.error(str(e))
            print(f"[rank {rank}] LoRA: {net.spec.total} adapter parameters over a frozen "
                  f"{net.base.spec.total}-parameter base ({a.lora_base or 'seeded genesis'})")
        eng = GenericFedEngine(cfg, net, shard, rank=rank, world=world, device=lr_)
    if a.resume:
        from .utils.checkpoint import load_checkpoint
        print(f"[rank {rank}] resumed:", load_checkpoint(a.resume, eng))

    log = RunLog(rank=rank)
    timer = PhaseTimer()
    t0 = time.time()
    for _ in range(a.rounds):
        with timer.phase("round"):
            eng.run_round()
        st = eng.read_state()
        acc = eng.evaluate(test) if rank == 0 else None        # sponsor (M:280-340)
        log.round(st["epoch"] - 1, st["global_loss"], test_acc=acc,
                  committee=[r for r, x in enumerate(st["roles"]) if x & 2])
        if cfg.dp_mode == 2 and rank == 0:
            eps, delta = eng.privacy_spent()
            print(f"epsilon {eps:.6g} delta {delta:g} epoch {st['epoch'] - 1}", flush=True)
        if cfg.dp_adaptive and rank == 0:
            _, clip, count = eng.last_update_norms(with_clip=True)
            print(f"clip {float(clip):.6g} noised unclipped count {float(count):.4g} next clip {eng.clip_now():.6g} "
                  f"epoch {st['epoch'] - 1}", flush=True)
        if cfg.dpsgd_on:
            eps, delta = eng.privacy_spent_local()
            print(f"[rank {rank}] local epsilon {eps:.6g} delta {delta:g} epoch {st['epoch'] - 1} (DP-SGD)",
                  flush=True)
    errs = eng.drain_blocks()
    summary = dict(rounds=a.rounds, wall_s=round(time.time() - t0, 3), timing=timer.summary(),
                   ledger_mismatches=errs, chain_ok=eng.host_ledger.verify_chain(),
                   blocks=eng.host_ledger.n_blocks(), symm=eng.heap.describe())
    if getattr(eng, "dpsgd", None) is not None:            # examples dropped for a non-finite gradient norm
        summary["dpsgd_dropped"] = int(eng.dpsgd.dropped.item())
    if getattr(eng, "poisson", None) is not None:          # the accounting and the capacity, never the sample
        eps, delta = eng.privacy_spent_local()
        summary["dpsgd_poisson"] = dict(epsilon=eps, delta=delta, cap=eng.poisson.cap,
                                        overflow_last_round=int(eng.poisson.overflow.item()))
    if getattr(eng, "grad_norms", None) is not None:        # gradient clipping: the last round's norms
        summary["grad_norms"] = [round(x, 6) for x in eng.grad_norms.tolist()]
        summary["skipped_steps"] = int(eng.skipped_steps.item())
    if a.checkpoint:
        from .utils.checkpoint import save_checkpoint
        summary["checkpoint"] = save_checkpoint(a.checkpoint, eng)
    if rank == 0:
        print("SUMMARY " + json.dumps(summary))
    if world > 1:
        torch.cuda.synchronize()
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
