"""Rounds/s of the other BASELINE.json configs (#3 LeNet-5 fp8, #4 ResNet-18 + one Byzantine
rank with committee 5, #5 BERT-base) on the generic engine.  One JSON line per config (rank 0).

  python -m torch.distributed.run --nnodes=1 --nproc-per-node=N --master-addr 127.0.0.1 \
      scripts/bench_models.py [--configs lenet5_fp8 resnet18_byz bert] [--rounds 6]

Timing: capture (1 eager round) + 2 warm-up rounds, then K rounds each bracketed by barrier +
synchronize and CUDA events on the engine stream, max over ranks; nvidia-smi clocks sampled
during the timed region.  Each line also carries the checks the protocol promises: replicas
bit-identical, host ledgers re-executed every election without mismatch, the Byzantine rank
never aggregated nor elected, and for the big models the achieved fraction of the NVLink
roofline of the FedAvg publish (bytes that must cross NVLink / 770 GB/s measured peer copy).
(The flagship number is bench.py; this covers model families.)
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch
import torch.distributed as dist

from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.data.synthetic import cifar_like, femnist_like, lm_corpus_like, tokens_like
from bflc_demo_b200.engine.generic import GenericFedEngine
from bflc_demo_b200.models.nets import build_model

CONFIGS = {
    #  name          model       dtype   samples batch  lr     bert_layers byzantine committee(8 GPUs)
    "mlp_fp8":      ("mlp",      "fp8",  4096,  512,   0.05,  0,  False, 3),
    "mlp_bf16":     ("mlp",      "bf16", 4096,  512,   0.05,  0,  False, 3),
    "lenet5_fp8":   ("lenet5",   "fp8",  2048,  128,   0.05,  0,  False, 3),
    "lenet5_bf16":  ("lenet5",   "bf16", 2048,  128,   0.05,  0,  False, 3),
    "resnet18_byz": ("resnet18", "bf16", 256,   64,    0.02,  0,  True,  5),   # BASELINE config #4
    "resnet18_gn":  ("resnet18", "bf16", 256,   64,    0.02,  0,  True,  5),   # config #4 with GroupNorm
    "bert":         ("bert",     "bf16", 32,    16,    0.002, 12, False, 3),
    "gpt":          ("gpt",      "bf16", 64,    16,    0.001, 12, False, 3),   # next-token, vocab 8192
    "bert_lora":    ("bert",     "bf16", 32,    16,    0.002, 12, False, 3),   # rank-8 adapters on q, v
    "gpt_lora":     ("gpt",      "bf16", 64,    16,    0.001, 12, False, 3),   # + the head
}
# LoRA configs: (rank, targets) of the adapters over the frozen base (models/lora.py); the update
# every round uploads, pulls and aggregates is the adapter vector
LORA = {"bert_lora": (8, "q,v"), "gpt_lora": (8, "q,v")}
# ResNet-18 norm of a config (default batch)
NORM = {"resnet18_gn": "group"}
NVLINK_GBS = 450.0   # H100 SXM NVLink 4 data-sheet rate, per direction per GPU (not a measurement)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="*", default=["mlp_fp8", "lenet5_fp8", "resnet18_byz", "bert"])
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--seq-len", type=int, default=128, help="bert config: token positions per sample")
    ap.add_argument("--min-seq-len", type=int, default=None,
                    help="bert config: shortest sample (default --seq-len); shorter ones are right-padded")
    ap.add_argument("--packed", action="store_true",
                    help="bert config: packed batches (every layer on the real tokens only)")
    ap.add_argument("--dropout", type=float, default=0.0,
                    help="bert config: training dropout probability in [0, 1) (default 0: none)")
    ap.add_argument("--optimizer", default="sgd", choices=["sgd", "adam"])
    from bflc_demo_b200.run import (add_aggregation_args, add_recipe_args, add_server_opt_args, check_seq_args,
                                    recipe_fields, server_opt_fields)
    add_recipe_args(ap)
    add_aggregation_args(ap)    # --total-steps defaults to every round a config runs (3 warm-up + --rounds)
    add_server_opt_args(ap)
    a = ap.parse_args()
    server = server_opt_fields(ap, a)
    if not 0.0 <= a.dropout < 1.0:
        ap.error(f"--dropout {a.dropout}: must lie in [0, 1)")
    seq_len, min_seq = check_seq_args(ap, a.seq_len, a.min_seq_len)
    padded = min_seq < seq_len or a.packed   # packed: token 0 is the pad id even at full length
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    lr_ = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(lr_)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", lr_))

    def sync():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()

    sys.path.insert(0, ROOT)
    from bench import ClockSampler

    for name in a.configs:
        model, dtype, S, B, lr, layers, byz, comm8 = CONFIGS[name]
        # committee: the BASELINE.json size at 8 GPUs (5 for config #4 -- larger than the trainer
        # set: re-election refills from the outgoing committee), scaled down on smaller boxes
        comm = comm8 if world == 8 else None
        byz_ranks = [world - 1] if (byz and world > 2) else []
        cfg = FLConfig.for_world(world, committee_size=comm, model=model, batch_size=B,
                                 samples_per_client=S, learning_rate=lr, dtype=dtype, ring_slots=256,
                                 byzantine_ranks=byz_ranks, optimizer=a.optimizer,
                                 aggregation=a.aggregation, trim=a.trim, **server,
                                 **recipe_fields(ap, a, (a.rounds + 3) * (S // B)),
                                 resnet_norm=NORM.get(name, "batch"),
                                 **(dict(lora_rank=LORA[name][0], lora_targets=LORA[name][1]) if name in LORA else {}))
        if model == "mlp":
            shard = femnist_like(world, S, seed=7, only=rank)[0]
        elif model in ("lenet5", "resnet18"):
            shard = cifar_like(world, S, seed=7, alpha=0.5)[rank]
        elif model == "gpt":
            shard = lm_corpus_like(world, S, seed=7, seq_len=seq_len, only=rank)[0]
        else:
            shard = tokens_like(world, S, seed=7, seq_len=seq_len, min_len=min_seq if padded else None)[rank]
        net = build_model(model, shard.n_classes, layers=layers or 12,
                          pad_id=0 if (model == "bert" and padded) else None,
                          packed=a.packed and model == "bert",
                          dropout=a.dropout if model in ("bert", "gpt") else 0.0, norm=cfg.resnet_norm)
        if cfg.lora_rank:
            from bflc_demo_b200.models.lora import lora_net_from_config
            net = lora_net_from_config(cfg, net)
        eng = GenericFedEngine(cfg, net, shard, rank=rank, world=world, device=lr_)
        eng.capture()
        for _ in range(2):
            eng.run_round()
        sync()
        sampler = ClockSampler(lr_) if rank == 0 else None
        if sampler:
            sampler.start()
        per_round, stamps = [], []
        for _ in range(a.rounds):
            sync()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(eng.stream):
                e0.record()
            eng.run_round()
            with torch.cuda.stream(eng.stream):
                e1.record()
            e1.synchronize()
            per_round.append(e0.elapsed_time(e1))
            stamps.append(eng.read_stamps())
        sync()
        clocks = sampler.stop() if sampler else None
        ms = torch.tensor(per_round, device="cuda", dtype=torch.float64)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        total_ms = float(ms.sum().item())
        st = eng.read_state()
        errs = eng.drain_blocks()
        blocks = eng.host_ledger.blocks()
        agg_us = sorted(s_["aggregate_publish_us"] for s_ in stamps)[len(stamps) // 2]
        agg = torch.tensor([agg_us], device="cuda", dtype=torch.float64)
        digs = [st["model_digest"]]
        all_errs = [errs]
        pkeys = sorted(stamps[0])
        pmed = torch.tensor([sorted(s_[k] for s_ in stamps)[len(stamps) // 2] for k in pkeys],
                            device="cuda", dtype=torch.float64)
        if world > 1:
            dist.all_reduce(pmed, op=dist.ReduceOp.MAX)
            dist.all_reduce(agg, op=dist.ReduceOp.MAX)
            digs = [None] * world
            dist.all_gather_object(digs, st["model_digest"])
            all_errs = [None] * world
            dist.all_gather_object(all_errs, errs)
        if rank == 0:
            P = int(net.spec.total)
            n_sel = max(len(b["selected"]) for b in blocks) if blocks else 0
            # bytes one rank must move over NVLink for the aggregation of a round
            if eng.two_shot:   # pull n_sel slices of P/n fp32, publish its slice (fp32 + bf16, x2 buffers) to n-1 peers
                nv_bytes = n_sel * P * 4 / world + (world - 1) * (P / world) * 12
            else:              # one-shot: pull n_sel whole fp32 uploads
                nv_bytes = n_sel * P * 4
            roof_us = nv_bytes / (NVLINK_GBS * 1e3)
            line = {
                "config": name, "model": model, "dtype": dtype, "n_gpus": world,
                "params": P, "upload_bytes_per_round": P * 4, "samples_per_client": S, "local_batch": B,
                **({"lora": {"rank": cfg.lora_rank, "targets": cfg.lora_targets,
                             "frozen_base_params": int(net.base.spec.total)}} if cfg.lora_rank else {}),
                "committee": cfg.committee_size, "trainers": cfg.n_trainers, "byzantine": cfg.byzantine_ranks,
                "rounds": a.rounds, "ms_per_round": total_ms / a.rounds, "optimizer": cfg.optimizer,
                **({"recipe": {k: getattr(cfg, k) for k in ("weight_decay", "lr_schedule", "warmup_steps",
                                                            "total_steps", "clip_grad_norm")},
                    "skipped_steps": (int(eng.skipped_steps.item()) if eng.skipped_steps is not None else None)}
                   if cfg.has_optim_recipe else {}),
                **({"seq_len": seq_len, "min_seq_len": min_seq, "packed": a.packed, "dropout": a.dropout}
                   if model == "bert" else {}),
                **({"seq_len": seq_len, "dropout": a.dropout, "vocab": net.n_classes} if model == "gpt" else {}),
                **({"resnet_norm": cfg.resnet_norm} if model == "resnet18" else {}),
                "rounds_per_s": a.rounds / (total_ms / 1e3), "global_loss": st["global_loss"],
                "graphs": {"train": eng.graph_train is not None, "validate": eng.graph_val is not None,
                           "capture_error": eng.capture_error},
                "two_shot": bool(eng.two_shot), "multicast": eng.heap.describe().get("multicast"),
                "replicas_bit_identical": len(set(digs)) == 1,
                "ledger_mismatches": [e for e in all_errs if e][:2], "chain_ok": eng.host_ledger.verify_chain(),
                "clocks": clocks,
                "phases_us_max_over_ranks": {k: round(v, 1) for k, v in zip(pkeys, pmed.tolist())},
                "fedavg": {"aggregate_publish_us_max_over_ranks": round(float(agg.item()), 1),
                           "nvlink_bytes_per_rank": int(nv_bytes), "roofline_us_at_770GBs": round(roof_us, 1),
                           "fraction_of_nvlink_roofline": round(roof_us / max(float(agg.item()), 1e-9), 3)},
            }
            if byz_ranks:
                bz = byz_ranks[0]
                as_tr = [b for b in blocks if bz in b["admitted"]]
                line["byzantine_check"] = {
                    "rank": bz, "rounds_as_trainer": len(as_tr),
                    "times_selected": sum(bz in b["selected"] for b in as_tr),
                    "ever_selected": any(bz in b["selected"] for b in blocks),
                    # with committee >= trainers every trainer is re-elected by construction
                    "ever_elected": any(b["role_after"][bz] == 2 for b in blocks),
                    "election_is_structural": cfg.committee_size >= cfg.n_trainers,
                    # per round the Byzantine rank trained: its median score vs the honest trainers'
                    # (block.median is per admitted trainer, in admission order)
                    "median_byz_vs_honest": [
                        [round(b["median"][b["admitted"].index(bz)], 4),
                         [round(m, 4) for t, m in zip(b["admitted"], b["median"]) if t != bz]]
                        for b in as_tr][:12]}
            print(json.dumps(line), flush=True)
        del eng
        torch.cuda.empty_cache()
        sync()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
