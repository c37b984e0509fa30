"""Multi-GPU protocol checks (run under torchrun, any world size 2..8). Rank 0 prints one
``RESULT {json}`` line.  Used by tests/test_gpu_multi.py.

Checks:
  fused       MLP fused engine: rounds advance, host ledgers verify, replicas bit-identical,
              committee rotates, loss falls
  byzantine   one sign-flipping rank is never aggregated nor elected
  two_shot    two-shot (slice-reduce + publish) aggregation gives the same digest as one-shot
  multicast   the same through NVLS multimem stores when the heap has a multicast mapping
  generic     LeNet-5 through the model-agnostic engine (validation on peers' HBM)
  lora        LoRA (rank 8 on q, v, ff1) over a frozen 2-layer GPT base: replicas bit-identical, base frozen
  lora_digest ranks given different LoRA bases: every rank refuses to build the engine
  dpsgd       DP-SGD LoRA GPT with per-rank secret noise keys: replicas bit-identical, ledgers agreeing,
              every rank's noise different
  dpsgd_full  the same with full-model DP-SGD on a 2-layer GPT (every parameter clipped and noised)
  dpsgd_conv  the same with DP-SGD on LeNet-5 (convolution sites, ``dpsgd_conv``)
  dpsgd_poisson  the "dpsgd" checks with Poisson sampling: every rank's secret sample different
  dpsgd_fused  the "dpsgd" checks with DP-SGD in the persistent MLP trainer (FusedEngine, ``dpsgd_fused``)
  gpt         a 2-layer GPT (causal attention, LM head) through the same engine: replicas bit-identical
              and ledgers agreeing after 3 captured rounds
  firstk      device-side first-K-wins admission (C:239-244): needed_updates = trainers - 1 and one
              artificially slow trainer -- every round completes with exactly K admitted, the
              straggler's update is dropped, the host ledger re-executes from the admitted mask
  fedavg      the aggregated global model is RIGHT, not just identical: after every round each rank
              recomputes sum_k w_k * upload_k (selected set + weights from the host ledger's block,
              uploads read out of the trainers' HBM, ascending rank order, fp32 fma) in PyTorch and
              compares it with the device result -- bf16 and fp8 engines
  robust      coordinate-wise median / trimmed mean with one Byzantine trainer and every admitted
              update selected: each round matches the reference recomputed from the trainers' HBM
              and stays inside the honest updates' range, one-shot and two-shot with multicast; a
              FedAvg control run leaves that range -- bf16 and fp8 engines
  serveropt   server optimizers (momentum, adam, yogi) on the median of every admitted update: each
              round the global model is the oracle step (protocol/oracle.py server_step) from the
              previous global model and the median recomputed from the trainers' HBM, and this
              rank's optimizer state matches the oracle's on the coordinates it reduces -- one-shot
              and two-shot with multicast, bf16 engine
  prox        FedProx local training (prox_mu > 0, Dirichlet(0.1) shards, Adam): every rank anchors its
              trainer at its own replica of the global model, which the peers' consensus rewrites -- the
              fused engine (bf16 and fp8) and the generic engine (LeNet-5 with a recipe) over three
              rounds: every replica's global model is bit-identical and every host ledger re-executes
              with no mismatch
  dp          differentially private FedAvg (clip 1, noise 0 and 0.8), two-shot with multicast, one
              Byzantine trainer at scale 1e3: each round the device norms are the sequential fp64 norms
              within 1 fp32 ulp, the global model is protocol/oracle.py dp_device_combine of the
              previous one bit for bit, the clip-only model moves at most C * sum w, and the replicas
              are bit-identical
"""
import os as _os, sys as _sys
_sys.path.insert(0, _os.path.dirname(_os.path.dirname(_os.path.abspath(__file__))))
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.data.synthetic import cifar_like, femnist_like


def main():
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); lr = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    which = sys.argv[1:] or ["fused", "byzantine", "two_shot", "generic"]
    out = {"world": world}

    def gather(x):
        box = [None] * world
        dist.all_gather_object(box, x)
        return box

    from bflc_demo_b200.engine.fused import FusedEngine

    def run_fused(rounds=6, **kw):
        kw.setdefault("dtype", os.environ.get("BFLC_CHECK_DTYPE", "bf16"))   # fp8: MXFP8 trainer + blobs
        cfg = FLConfig.for_world(world, hidden=256, batch_size=128, samples_per_client=512,
                                 learning_rate=0.05, **kw)
        shard = femnist_like(world, 512, seed=3, only=rank)[0]
        eng = FusedEngine(cfg, shard, rank=rank, world=world, device=lr)
        eng.capture()
        hist = [eng.run_round_e2e() for _ in range(rounds)]
        errs = eng.drain_blocks()
        st = eng.read_state()
        info = dict(epoch=st["epoch"], digest=st["model_digest"], errs=errs,
                    chain=eng.host_ledger.verify_chain(), blocks=eng.host_ledger.n_blocks(),
                    last_hash=eng.host_ledger.blocks()[-1]["hash"], loss=[h["global_loss"] for h in hist],
                    roles=[h["roles"] for h in hist], symm=eng.heap.describe())
        blocks = eng.host_ledger.blocks()
        torch.cuda.synchronize(); dist.barrier()   # nobody may still be reading my heap
        del eng
        torch.cuda.synchronize(); dist.barrier()
        return info, blocks

    if "fused" in which:
        info, blocks = run_fused()
        allinfo = gather(info)
        out["fused"] = dict(
            epochs=[i["epoch"] for i in allinfo], errs=sum((i["errs"] for i in allinfo), []),
            identical_digest=len({i["digest"] for i in allinfo}) == 1,
            identical_chain=len({i["last_hash"] for i in allinfo}) == 1,
            chain_ok=all(i["chain"] for i in allinfo), loss=info["loss"],
            committee_rotates=len({tuple(r) for r in info["roles"]}) > 1 if world > 2 else True,
            symm=info["symm"])
    if "byzantine" in which and world >= 4:
        byz = world - 1
        info, blocks = run_fused(rounds=6, byzantine_ranks=[byz], byzantine_scale=5.0)
        sel = [b["selected"] for b in blocks]
        elected = [b["role_after"][byz] for b in blocks]
        admitted = [byz in b["admitted"] for b in blocks]
        out["byzantine"] = dict(rank=byz, ever_selected=any(byz in s for s in sel),
                                ever_elected=any(e == 2 for e in elected),
                                times_admitted=sum(admitted),
                                median_of_byz=[b["median"][b["admitted"].index(byz)] for b in blocks if byz in b["admitted"]][:3],
                                median_best=[max(b["median"]) for b in blocks][:3])
    if "two_shot" in which:
        # (local training uses split-K atomics, so two separate runs are not bit-comparable;
        #  what must hold in every mode is that all replicas of one run are bit-identical)
        res = {}
        for name, kw in (("two_shot_p2p", dict(two_shot=True, use_multicast=False)),
                         ("two_shot_multicast", dict(two_shot=True, use_multicast=True))):
            r, _ = run_fused(rounds=4, **kw)
            g = gather(r)
            res[name] = dict(identical=len({i["digest"] for i in g}) == 1,
                             errs=sum((i["errs"] for i in g), []), chain_ok=all(i["chain"] for i in g),
                             loss=r["loss"], multicast=r["symm"]["multicast"],
                             multicast_error=r["symm"]["multicast_error"], notes=r["symm"]["notes"])
        out["two_shot"] = res
    if "firstk" in which and world >= 4:
        res = {}
        slow = world - 1
        for dt in ("bf16", "fp8"):
            base = FLConfig.for_world(world)
            k = base.n_trainers - 1
            cfg = FLConfig.for_world(world, needed_updates=k, hidden=256, batch_size=128,
                                     samples_per_client=512, learning_rate=0.05, dtype=dt,
                                     straggler_ranks=[slow], straggler_delay_us=400)
            shard = femnist_like(world, 512, seed=3, only=rank)[0]
            eng = FusedEngine(cfg, shard, rank=rank, world=world, device=lr)
            eng.capture()
            for _ in range(6):
                eng.run_round()
            errs = eng.drain_blocks()
            st = eng.read_state()
            blocks = eng.host_ledger.blocks()
            g = gather(dict(digest=st["model_digest"], errs=errs, epoch=st["epoch"]))
            res[dt] = dict(k=k, trainers=cfg.n_trainers, epoch=st["epoch"],
                           admitted_per_round=[len(b["admitted"]) for b in blocks],
                           slow_rank=slow, slow_was_trainer=sum(b["role_before"][slow] == 1 for b in blocks),
                           slow_admitted=sum(slow in b["admitted"] for b in blocks),
                           identical=len({i["digest"] for i in g}) == 1,
                           errs=sum((i["errs"] for i in g), []), chain_ok=eng.host_ledger.verify_chain())
            torch.cuda.synchronize(); dist.barrier()
            del eng
            torch.cuda.synchronize(); dist.barrier()
        out["firstk"] = res
    if "fedavg" in which:
        res = {}
        for dt in ("bf16", "fp8"):
            cfg = FLConfig.for_world(world, hidden=256, batch_size=128, samples_per_client=512,
                                     learning_rate=0.05, dtype=dt)
            shard = femnist_like(world, 512, seed=3, only=rank)[0]
            eng = FusedEngine(cfg, shard, rank=rank, world=world, device=lr)
            eng.capture()
            o, P = eng.layout.offsets, eng.n_params
            worst, exact, errs = 0.0, True, []
            for _ in range(4):
                eng.run_round()
                torch.cuda.synchronize(); dist.barrier()
                errs += eng.drain_blocks()
                blk = eng.host_ledger.blocks()[-1]
                par = blk["epoch"] & 1
                ref = torch.zeros(P, device="cuda", dtype=torch.float64)
                for t, w in zip(blk["selected"], blk["weight"]):
                    up = eng.heap.view(o[f"upload_master{par}"], [P], torch.float32, rank=t)
                    # fp32 fma(w, v, acc): the product is exact in fp64, one rounding back to fp32
                    ref = (ref + up.double() * float(w)).float().double()
                d = (eng.global_master.double() - ref).abs().max().item()
                worst = max(worst, d / max(ref.abs().max().item(), 1e-30))
                exact = exact and bool((eng.global_master.double() == ref).all())
                torch.cuda.synchronize(); dist.barrier()
            g = gather(dict(worst=worst, exact=exact, errs=errs, n_sel=len(blk["selected"])))
            res[dt] = dict(worst_rel=max(i["worst"] for i in g), bit_exact=all(i["exact"] for i in g),
                           errs=sum((i["errs"] for i in g), []), n_selected=g[0]["n_sel"])
            torch.cuda.synchronize(); dist.barrier()
            del eng
            torch.cuda.synchronize(); dist.barrier()
        out["fedavg"] = res
    if "robust" in which and world >= 4:
        # Byzantine-robust aggregation: every admitted update selected (aggregate_count = trainers),
        # one byz_mode=1 trainer.  Each round the new global model must be the reference recomputed
        # from the selected trainers' HBM (bit for bit outside NaN) and stay inside the honest
        # updates' range; a FedAvg control run leaves that range.
        from bflc_demo_b200.protocol.oracle import aggregation_trim, robust_combine
        byz = world - 1
        comm = 1 if world == 4 else None
        rules = [("fedavg", 1), ("median", 1)] + ([("trimmed_mean", 1)] if world >= 8 else [])
        res = {}
        for dt in ("bf16", "fp8"):
            for rule, trim in rules:
                for mode, kw in (("one_shot", dict(two_shot=False)),
                                 ("two_shot_mc", dict(two_shot=True, use_multicast=True))):
                    if rule == "fedavg" and mode != "one_shot":
                        continue
                    base = FLConfig.for_world(world, committee_size=comm)
                    cfg = FLConfig.for_world(world, committee_size=comm, aggregate_count=base.n_trainers,
                                             hidden=256, batch_size=128, samples_per_client=512,
                                             learning_rate=0.05, dtype=dt, byzantine_ranks=[byz],
                                             byzantine_scale=5.0, aggregation=rule, trim=trim, **kw)
                    shard = femnist_like(world, 512, seed=3, only=rank)[0]
                    eng = FusedEngine(cfg, shard, rank=rank, world=world, device=lr)
                    eng.capture()
                    o, P = eng.layout.offsets, eng.n_params
                    exact, inside, byz_rounds, errs = True, True, 0, []
                    for _ in range(4):
                        eng.run_round()
                        torch.cuda.synchronize(); dist.barrier()
                        errs += eng.drain_blocks()
                        blk = eng.host_ledger.blocks()[-1]
                        par = blk["epoch"] & 1
                        ups = {t: eng.heap.view(o[f"upload_master{par}"], [P], torch.float32, rank=t).cpu().numpy()
                               for t in blk["selected"]}
                        got = eng.global_master.cpu().numpy()
                        vals = np.stack([ups[t] for t in blk["selected"]])
                        if rule == "fedavg":
                            ref = np.zeros(P, np.float32)
                            for t, w in zip(blk["selected"], blk["weight"]):
                                ref = (ref.astype(np.float64) + ups[t].astype(np.float64) * float(w)).astype(np.float32)
                        else:
                            ref = robust_combine(vals, aggregation_trim(rule, trim))
                        exact = exact and bool(((got.view(np.uint32) == ref.view(np.uint32))
                                                | (np.isnan(got) & np.isnan(ref))).all())
                        honest = [ups[t] for t in blk["selected"] if t != byz]
                        if byz in blk["selected"] and len(honest) >= 2:
                            byz_rounds += 1
                            h = np.stack(honest)
                            inside = inside and bool(((got >= h.min(0)) & (got <= h.max(0))).all())
                        torch.cuda.synchronize(); dist.barrier()
                    st = eng.read_state()
                    g = gather(dict(exact=exact, inside=inside, errs=errs, digest=st["model_digest"],
                                    byz_rounds=byz_rounds))
                    res[f"{dt}_{rule}{trim if rule == 'trimmed_mean' else ''}_{mode}"] = dict(
                        bit_exact=all(i["exact"] for i in g), inside_honest=all(i["inside"] for i in g),
                        byz_rounds=min(i["byz_rounds"] for i in g), identical=len({i["digest"] for i in g}) == 1,
                        errs=sum((i["errs"] for i in g), []), multicast=eng.heap.has_multicast)
                    torch.cuda.synchronize(); dist.barrier()
                    del eng
                    torch.cuda.synchronize(); dist.barrier()
        out["robust"] = res
    if "serveropt" in which and world >= 4:
        from bflc_demo_b200.protocol.oracle import robust_combine, server_step
        comm = 1 if world == 4 else None
        res = {}
        for opt in ("momentum", "adam", "yogi"):
            for mode, kw in (("one_shot", dict(two_shot=False)),
                             ("two_shot_mc", dict(two_shot=True, use_multicast=True))):
                base = FLConfig.for_world(world, committee_size=comm)
                cfg = FLConfig.for_world(world, committee_size=comm, aggregate_count=base.n_trainers,
                                         hidden=256, batch_size=128, samples_per_client=512,
                                         learning_rate=0.05, aggregation="median", server_opt=opt, **kw)
                shard = femnist_like(world, 512, seed=3, only=rank)[0]
                eng = FusedEngine(cfg, shard, rank=rank, world=world, device=lr)
                o, P = eng.layout.offsets, eng.n_params
                # the two-shot slice this rank reduces (k_consensus: even float4 slices)
                nv = P // 4
                per = (nv + world - 1) // world
                per += per & 1
                lo = min(per * rank, nv)
                lo, hi = (4 * lo, 4 * min(lo + per, nv)) if eng.two_shot else (0, P)
                g = eng.global_master.cpu().numpy()
                m, v = np.zeros(P, np.float32), np.zeros(P, np.float32)
                exact, state_exact, errs = True, True, []
                for i in range(4):
                    if i == 0:
                        eng.capture()        # the warm-up is a real round
                    else:
                        eng.run_round()
                    torch.cuda.synchronize(); dist.barrier()
                    errs += eng.drain_blocks()
                    blk = eng.host_ledger.blocks()[-1]
                    par = blk["epoch"] & 1
                    vals = np.stack([eng.heap.view(o[f"upload_master{par}"], [P], torch.float32, rank=t).cpu().numpy()
                                     for t in blk["selected"]])
                    g, m, v = server_step(g, robust_combine(vals, 1 << 30), m, v, opt, cfg.server_opt_constants)
                    got = eng.global_master.cpu().numpy()
                    exact = exact and bool(((got.view(np.uint32) == g.view(np.uint32)) | (np.isnan(got) & np.isnan(g))).all())
                    for t, want in zip(eng.server_state, (m, v)):
                        s = t.cpu().numpy()[lo:hi]
                        state_exact = state_exact and bool(((s.view(np.uint32) == want[lo:hi].view(np.uint32))
                                                            | (np.isnan(s) & np.isnan(want[lo:hi]))).all())
                    torch.cuda.synchronize(); dist.barrier()
                st = eng.read_state()
                gg = gather(dict(exact=exact, state_exact=state_exact, errs=errs, digest=st["model_digest"]))
                res[f"{opt}_{mode}"] = dict(
                    bit_exact=all(i["exact"] for i in gg), state_exact=all(i["state_exact"] for i in gg),
                    identical=len({i["digest"] for i in gg}) == 1, errs=sum((i["errs"] for i in gg), []),
                    two_shot=eng.two_shot, multicast=eng.heap.has_multicast)
                torch.cuda.synchronize(); dist.barrier()
                del eng
                torch.cuda.synchronize(); dist.barrier()
        out["serveropt"] = res
    if "dp" in which:
        # differentially private FedAvg, two-shot with multicast, one Byzantine trainer at scale 1e3: each
        # round the global model is protocol/oracle.py dp_device_combine of the previous one and the
        # selected uploads read out of the trainers' HBM, fed with the device's own norms, and the
        # replicas are bit-identical
        from bflc_demo_b200.protocol.oracle import dp_device_combine, dp_norm
        byz = world - 1
        res = {}
        for noise in (0.0, 0.8):
            cfg = FLConfig.for_world(world, hidden=256, batch_size=128, samples_per_client=512,
                                     learning_rate=0.05, two_shot=True, use_multicast=True, byzantine_ranks=[byz],
                                     byzantine_scale=1e3, dp_clip=1.0, dp_noise=noise, dp_seed=0xD15EA5E)
            shard = femnist_like(world, 512, seed=3, only=rank)[0]
            eng = FusedEngine(cfg, shard, rank=rank, world=world, device=lr)
            o, P = eng.layout.offsets, eng.n_params
            g = eng.global_master.cpu().numpy()
            exact, norms_ok, bounded, errs, max_move = True, True, True, [], 0.0
            for i in range(4):
                if i == 0:
                    eng.capture()
                else:
                    eng.run_round()
                torch.cuda.synchronize(); dist.barrier()
                errs += eng.drain_blocks()
                blk = eng.host_ledger.blocks()[-1]
                par = blk["epoch"] & 1
                norms = eng.last_update_norms()
                vals = np.stack([eng.heap.view(o[f"upload_master{par}"], [P], torch.float32, rank=t).cpu().numpy()
                                 for t in blk["selected"]])
                for t, u in zip(blk["selected"], vals):
                    ref = dp_norm((u - g).astype(np.float32))
                    norms_ok = norms_ok and abs(float(norms[t]) - float(ref)) <= float(np.spacing(ref))
                want = dp_device_combine(g, vals, blk["weight"], [norms[t] for t in blk["selected"]], "fedavg", 1,
                                         1.0, noise, cfg.dp_seed, blk["epoch"])
                got = eng.global_master.cpu().numpy()
                exact = exact and bool(((got.view(np.uint32) == want.view(np.uint32))
                                        | (np.isnan(got) & np.isnan(want))).all())
                move = float(np.linalg.norm(got.astype(np.float64) - g))
                max_move = max(max_move, move)
                if noise == 0.0:   # |g' - g| <= C * sum w (+ rounding relative to |g|)
                    bounded = bounded and move <= 1.0 * sum(blk["weight"]) * (1 + 1e-5) + 1e-5 * (
                        1 + float(np.linalg.norm(g)))
                g = got
                torch.cuda.synchronize(); dist.barrier()
            st = eng.read_state()
            gg = gather(dict(exact=exact, norms_ok=norms_ok, bounded=bounded, errs=errs, digest=st["model_digest"]))
            res[f"noise{noise}"] = dict(
                bit_exact=all(i["exact"] for i in gg), norms_ok=all(i["norms_ok"] for i in gg),
                bounded=all(i["bounded"] for i in gg), identical=len({i["digest"] for i in gg}) == 1,
                errs=sum((i["errs"] for i in gg), []), max_move=max_move, two_shot=eng.two_shot,
                multicast=eng.heap.has_multicast, launches_per_round=eng.launches_per_round)
            torch.cuda.synchronize(); dist.barrier()
            del eng
            torch.cuda.synchronize(); dist.barrier()
        out["dp"] = res
    if "dp_adaptive" in which:
        # adaptive clipping, two-shot with multicast, from a clip 100x too small: each round the clip record
        # (C_t, b~, n_sel) is oracle.dp_clip_round's from the device's own norms, the model is
        # dp_device_combine's at C_t, the ledger re-executes the clip step, and the replicas are bit-identical
        from bflc_demo_b200.protocol.oracle import dp_clip_round, dp_device_combine
        res = {}
        for noise in (0.0, 0.8):
            cfg = FLConfig.for_world(world, hidden=256, batch_size=128, samples_per_client=512,
                                     learning_rate=0.05, two_shot=True, use_multicast=True, dp_clip=0.01,
                                     dp_noise=noise, dp_seed=0xD15EA5E, dp_clip_quantile=0.5, dp_clip_lr=0.5,
                                     dp_count_noise=1.0 if noise else 0.0)
            q, clr, sb = (float(x) for x in cfg.dp_adapt_constants)
            shard = femnist_like(world, 512, seed=3, only=rank)[0]
            eng = FusedEngine(cfg, shard, rank=rank, world=world, device=lr)
            o, P = eng.layout.offsets, eng.n_params
            g = eng.global_master.cpu().numpy()
            clip = np.float32(eng.clip_now())
            exact, clip_ok, errs, clips = True, True, [], [float(clip)]
            for i in range(6):
                if i == 0:
                    eng.capture()
                else:
                    eng.run_round()
                torch.cuda.synchronize(); dist.barrier()
                errs += eng.drain_blocks()
                blk = eng.host_ledger.blocks()[-1]
                par = blk["epoch"] & 1
                norms, c_dev, b_dev = eng.last_update_norms(with_clip=True)
                sel_norms = [norms[t] for t in blk["selected"]]
                count, nxt = dp_clip_round(sel_norms, clip, q, clr, sb, cfg.dp_seed, blk["epoch"])
                clip_ok = clip_ok and c_dev == clip and b_dev == count and np.float32(eng.clip_now()) == nxt
                vals = np.stack([eng.heap.view(o[f"upload_master{par}"], [P], torch.float32, rank=t).cpu().numpy()
                                 for t in blk["selected"]])
                want = dp_device_combine(g, vals, blk["weight"], sel_norms, "fedavg", 1, clip, noise, cfg.dp_seed,
                                         blk["epoch"], count_noise=sb)
                got = eng.global_master.cpu().numpy()
                exact = exact and bool(((got.view(np.uint32) == want.view(np.uint32))
                                        | (np.isnan(got) & np.isnan(want))).all())
                g, clip = got, nxt
                clips.append(float(clip))
                torch.cuda.synchronize(); dist.barrier()
            st = eng.read_state()
            gg = gather(dict(exact=exact, clip_ok=clip_ok, errs=errs, digest=st["model_digest"], clip=clips[-1]))
            res[f"noise{noise}"] = dict(
                bit_exact=all(i["exact"] for i in gg), clip_ok=all(i["clip_ok"] for i in gg),
                identical=len({i["digest"] for i in gg}) == 1 and len({i["clip"] for i in gg}) == 1,
                errs=sum((i["errs"] for i in gg), []), clips=clips, two_shot=eng.two_shot,
                multicast=eng.heap.has_multicast)
            torch.cuda.synchronize(); dist.barrier()
            del eng
            torch.cuda.synchronize(); dist.barrier()
        out["dp_adaptive"] = res
    if "prox" in which:
        import hashlib
        from bflc_demo_b200.engine.generic import GenericFedEngine
        from bflc_demo_b200.models.nets import LeNet5
        res = {}
        for name in ("fused_bf16", "fused_fp8", "generic_lenet5"):
            if name.startswith("fused"):
                cfg = FLConfig.for_world(world, hidden=256, batch_size=128, samples_per_client=512, learning_rate=0.05,
                                         optimizer="adam", dtype=name[6:], prox_mu=0.05, non_iid_alpha=0.1)
                eng = FusedEngine(cfg, femnist_like(world, 512, seed=3, only=rank, alpha=0.1)[0],
                                  rank=rank, world=world, device=lr)
                anchored = eng.trainer.anchor is eng.global_master
                eng.capture()
                for _ in range(2):
                    eng.run_round_e2e()
            else:
                cfg = FLConfig.for_world(world, batch_size=64, samples_per_client=256, learning_rate=0.05,
                                         model="lenet5", dataset="cifar10", optimizer="adam", prox_mu=0.05,
                                         non_iid_alpha=0.1, weight_decay=0.01, clip_grad_norm=1.0)
                eng = GenericFedEngine(cfg, LeNet5(10), cifar_like(world, 256, seed=2, alpha=0.1)[rank],
                                       rank=rank, world=world, device=lr)
                anchored = eng.recipe_step.anchor is eng.global_master
                eng.capture()
                for _ in range(2):
                    eng.run_round()
            errs = eng.drain_blocks()
            st = eng.read_state()
            torch.cuda.synchronize(); dist.barrier()   # every rank's last publish has landed in every replica
            h = hashlib.sha256(eng.global_master.cpu().numpy().tobytes()).hexdigest()
            g = gather(dict(h=h, digest=st["model_digest"], errs=errs, epoch=st["epoch"], anchored=anchored,
                            chain=eng.host_ledger.verify_chain()))
            res[name] = dict(identical=len({i["h"] for i in g}) == 1 and len({i["digest"] for i in g}) == 1,
                             errs=sum((i["errs"] for i in g), []), epochs=[i["epoch"] for i in g],
                             anchored=all(i["anchored"] for i in g), chain_ok=all(i["chain"] for i in g))
            torch.cuda.synchronize(); dist.barrier()
            del eng
            torch.cuda.synchronize(); dist.barrier()
        out["prox"] = res
    if "generic" in which:
        from bflc_demo_b200.engine.generic import GenericFedEngine
        from bflc_demo_b200.models.nets import LeNet5
        cfg = FLConfig.for_world(world, batch_size=64, samples_per_client=256, learning_rate=0.05,
                                 model="lenet5", dataset="cifar10")
        shard = cifar_like(world, 256, seed=2)[rank]
        eng = GenericFedEngine(cfg, LeNet5(10), shard, rank=rank, world=world, device=lr)
        acc0 = eng.evaluate(shard)
        for _ in range(5):
            eng.run_round()
        errs = eng.drain_blocks()
        st = eng.read_state()
        g = gather(dict(digest=st["model_digest"], errs=errs, epoch=st["epoch"]))
        out["generic_lenet5"] = dict(epoch=st["epoch"], acc_before=acc0, acc_after=eng.evaluate(shard),
                                     identical=len({i["digest"] for i in g}) == 1,
                                     errs=sum((i["errs"] for i in g), []), loss=st["global_loss"])
        torch.cuda.synchronize(); dist.barrier()
        del eng
        torch.cuda.synchronize(); dist.barrier()
    if "gpt" in which:
        # a 2-layer GPT (causal attention, vocabulary-wide cross-entropy) through the generic engine:
        # replicas stay bit-identical and every host ledger agrees with the device's
        from bflc_demo_b200.data.synthetic import lm_corpus_like
        from bflc_demo_b200.engine.generic import GenericFedEngine
        from bflc_demo_b200.models.nets import GPT
        cfg = FLConfig.for_world(world, batch_size=16, samples_per_client=64, learning_rate=1e-3, model="gpt",
                                 optimizer="adam")
        shard = lm_corpus_like(world, 64, seed=2, seq_len=128, only=rank)[0]
        eng = GenericFedEngine(cfg, GPT(layers=2), shard, rank=rank, world=world, device=lr)
        eng.capture()
        for _ in range(3):
            eng.run_round()
        errs = eng.drain_blocks()
        st = eng.read_state()
        g = gather(dict(digest=st["model_digest"], errs=errs, epoch=st["epoch"], chain=eng.host_ledger.verify_chain()))
        out["gpt"] = dict(epoch=st["epoch"], identical=len({i["digest"] for i in g}) == 1,
                          errs=sum((i["errs"] for i in g), []), chain_ok=all(i["chain"] for i in g),
                          loss=st["global_loss"], graphs=eng.graph_train is not None)
        torch.cuda.synchronize(); dist.barrier()
        del eng
        torch.cuda.synchronize(); dist.barrier()
    if "lora" in which:
        # LoRA on a 2-layer GPT: the update is the adapter vector over a frozen base every rank holds;
        # replicas stay bit-identical, the base never moves and every host ledger agrees with the device's
        from bflc_demo_b200.data.synthetic import lm_corpus_like
        from bflc_demo_b200.engine.generic import GenericFedEngine
        from bflc_demo_b200.models.lora import lora_net_from_config
        from bflc_demo_b200.models.nets import GPT
        cfg = FLConfig.for_world(world, batch_size=16, samples_per_client=64, learning_rate=2e-3, model="gpt",
                                 optimizer="adam", lora_rank=8, lora_targets="q,v,ff1")
        shard = lm_corpus_like(world, 64, seed=2, seq_len=128, only=rank)[0]
        net = lora_net_from_config(cfg, GPT(layers=2))
        eng = GenericFedEngine(cfg, net, shard, rank=rank, world=world, device=lr)
        base0 = net.base_buffers(eng.dev)[0].clone()
        eng.capture()
        for _ in range(3):
            eng.run_round()
        errs = eng.drain_blocks()
        st = eng.read_state()
        base_same = bool(torch.equal(net.base_buffers(eng.dev)[0], base0))
        g = gather(dict(digest=st["model_digest"], errs=errs, epoch=st["epoch"], chain=eng.host_ledger.verify_chain(),
                        base_same=base_same, base_digest=eng.base_digest))
        out["lora"] = dict(epoch=st["epoch"], identical=len({i["digest"] for i in g}) == 1,
                           errs=sum((i["errs"] for i in g), []), chain_ok=all(i["chain"] for i in g),
                           base_frozen=all(i["base_same"] for i in g),
                           one_base=len({i["base_digest"] for i in g}) == 1, n_params=eng.n_params,
                           adapters=net.spec.total, loss=st["global_loss"], graphs=eng.graph_train is not None)
        torch.cuda.synchronize(); dist.barrier()
        del eng
        torch.cuda.synchronize(); dist.barrier()
    if "dpsgd" in which:
        # DP-SGD LoRA GPT with each rank's own secret noise key: replicas stay bit-identical, every host
        # ledger agrees with the device's, and no two ranks draw the same noise
        import hashlib

        from bflc_demo_b200._native import C
        from bflc_demo_b200.data.synthetic import lm_corpus_like
        from bflc_demo_b200.engine.generic import GenericFedEngine
        from bflc_demo_b200.models.lora import lora_net_from_config
        from bflc_demo_b200.models.nets import GPT
        cfg = FLConfig.for_world(world, batch_size=16, samples_per_client=64, learning_rate=2e-3, model="gpt",
                                 optimizer="adam", lora_rank=8, dpsgd_clip=1.0, dpsgd_noise=1.0)
        shard = lm_corpus_like(world, 64, seed=2, seq_len=128, only=rank)[0]
        eng = GenericFedEngine(cfg, lora_net_from_config(cfg, GPT(layers=2)), shard, rank=rank, world=world,
                               device=lr)
        eng.capture()
        for _ in range(3):
            eng.run_round()
        errs = eng.drain_blocks()
        st = eng.read_state()
        noise = torch.zeros(1024, device=eng.dev)
        C().dpsgd_noise(noise, eng.dpsgd_seed, eng.opt_step_word, 0, 1.0)
        g = gather(dict(digest=st["model_digest"], errs=errs, chain=eng.host_ledger.verify_chain(),
                        noise=hashlib.sha256(noise.cpu().numpy().tobytes()).hexdigest()))
        out["dpsgd"] = dict(epoch=st["epoch"], identical=len({i["digest"] for i in g}) == 1,
                            errs=sum((i["errs"] for i in g), []), chain_ok=all(i["chain"] for i in g),
                            noise_distinct=len({i["noise"] for i in g}) == len(g), graphs=eng.graph_train is not None)
        torch.cuda.synchronize(); dist.barrier()
        del eng
        torch.cuda.synchronize(); dist.barrier()
    if "dpsgd_full" in which:
        # full-model DP-SGD on a 2-layer GPT: the same three checks as "dpsgd"
        import hashlib

        from bflc_demo_b200._native import C
        from bflc_demo_b200.data.synthetic import lm_corpus_like
        from bflc_demo_b200.engine.generic import GenericFedEngine
        from bflc_demo_b200.models.nets import GPT
        cfg = FLConfig.for_world(world, batch_size=16, samples_per_client=64, learning_rate=2e-3, model="gpt",
                                 optimizer="adam", dpsgd_clip=1.0, dpsgd_noise=1.0, dpsgd_full_model=True)
        shard = lm_corpus_like(world, 64, seed=2, seq_len=128, only=rank)[0]
        eng = GenericFedEngine(cfg, GPT(layers=2), shard, rank=rank, world=world, device=lr)
        eng.capture()
        for _ in range(3):
            eng.run_round()
        errs = eng.drain_blocks()
        st = eng.read_state()
        noise = torch.zeros(1024, device=eng.dev)
        C().dpsgd_noise(noise, eng.dpsgd_seed, eng.opt_step_word, 0, 1.0)
        g = gather(dict(digest=st["model_digest"], errs=errs, chain=eng.host_ledger.verify_chain(),
                        noise=hashlib.sha256(noise.cpu().numpy().tobytes()).hexdigest()))
        out["dpsgd_full"] = dict(epoch=st["epoch"], identical=len({i["digest"] for i in g}) == 1,
                                 errs=sum((i["errs"] for i in g), []), chain_ok=all(i["chain"] for i in g),
                                 noise_distinct=len({i["noise"] for i in g}) == len(g),
                                 graphs=eng.graph_train is not None)
        torch.cuda.synchronize(); dist.barrier()
        del eng
        torch.cuda.synchronize(); dist.barrier()
    if "dpsgd_poisson" in which:
        # the "dpsgd" case with Poisson sampling: replicas bit-identical, ledgers agreeing, and every rank's
        # sample (compared by digest here only; it never leaves the rank otherwise) its own
        import hashlib

        from bflc_demo_b200.data.synthetic import lm_corpus_like
        from bflc_demo_b200.engine.generic import GenericFedEngine
        from bflc_demo_b200.models.lora import lora_net_from_config
        from bflc_demo_b200.models.nets import GPT
        cfg = FLConfig.for_world(world, batch_size=16, samples_per_client=64, learning_rate=2e-3, model="gpt",
                                 optimizer="adam", lora_rank=8, dpsgd_clip=1.0, dpsgd_noise=1.0,
                                 dpsgd_sampling="poisson")
        shard = lm_corpus_like(world, 64, seed=2, seq_len=128, only=rank)[0]
        eng = GenericFedEngine(cfg, lora_net_from_config(cfg, GPT(layers=2)), shard, rank=rank, world=world,
                               device=lr)
        eng.capture()
        for _ in range(3):
            eng.run_round()
        errs = eng.drain_blocks()
        st = eng.read_state()
        g = gather(dict(digest=st["model_digest"], errs=errs, chain=eng.host_ledger.verify_chain(),
                        sample=hashlib.sha256(eng.poisson.idx.cpu().numpy().tobytes()).hexdigest()))
        out["dpsgd_poisson"] = dict(epoch=st["epoch"], identical=len({i["digest"] for i in g}) == 1,
                                    errs=sum((i["errs"] for i in g), []), chain_ok=all(i["chain"] for i in g),
                                    sample_distinct=len({i["sample"] for i in g}) == len(g),
                                    graphs=eng.graph_train is not None)
        torch.cuda.synchronize(); dist.barrier()
        del eng
        torch.cuda.synchronize(); dist.barrier()
    if "dpsgd_conv" in which:
        # DP-SGD on LeNet-5's convolutions and linear layers: the same three checks as "dpsgd"
        import hashlib

        from bflc_demo_b200._native import C
        from bflc_demo_b200.data.synthetic import cifar_like
        from bflc_demo_b200.engine.generic import GenericFedEngine
        from bflc_demo_b200.models.nets import LeNet5
        cfg = FLConfig.for_world(world, batch_size=32, samples_per_client=128, learning_rate=0.02, model="lenet5",
                                 dpsgd_clip=1.0, dpsgd_noise=1.0, dpsgd_conv=True)
        shard = cifar_like(world, 128, seed=2)[rank]
        eng = GenericFedEngine(cfg, LeNet5(), shard, rank=rank, world=world, device=lr)
        eng.capture()
        for _ in range(3):
            eng.run_round()
        errs = eng.drain_blocks()
        st = eng.read_state()
        noise = torch.zeros(1024, device=eng.dev)
        C().dpsgd_noise(noise, eng.dpsgd_seed, eng.opt_step_word, 0, 1.0)
        g = gather(dict(digest=st["model_digest"], errs=errs, chain=eng.host_ledger.verify_chain(),
                        noise=hashlib.sha256(noise.cpu().numpy().tobytes()).hexdigest()))
        out["dpsgd_conv"] = dict(epoch=st["epoch"], identical=len({i["digest"] for i in g}) == 1,
                                 errs=sum((i["errs"] for i in g), []), chain_ok=all(i["chain"] for i in g),
                                 noise_distinct=len({i["noise"] for i in g}) == len(g),
                                 graphs=eng.graph_train is not None)
        torch.cuda.synchronize(); dist.barrier()
        del eng
        torch.cuda.synchronize(); dist.barrier()
    if "dpsgd_fused" in which:
        # DP-SGD in the persistent MLP trainer with each rank's own secret noise key: the same checks as "dpsgd"
        import hashlib

        from bflc_demo_b200._native import C
        from bflc_demo_b200.engine.fused import FusedEngine
        cfg = FLConfig.for_world(world, model="mlp", batch_size=256, samples_per_client=1024, learning_rate=0.05,
                                 optimizer="adam", dpsgd_clip=0.5, dpsgd_noise=1.0, dpsgd_fused=True)
        eng = FusedEngine(cfg, femnist_like(world, 1024, seed=7, only=rank)[0], rank=rank, world=world, device=lr)
        eng.capture()
        for _ in range(3):
            eng.run_round()
        torch.cuda.synchronize()
        errs = eng.drain_blocks()
        st = eng.read_state()
        noise = torch.zeros(1024, device=eng.dev)
        C().dpsgd_noise(noise, eng.dpsgd_seed, torch.zeros(1, device=eng.dev, dtype=torch.int32), 0, 1.0)
        g = gather(dict(digest=st["model_digest"], errs=errs, chain=eng.host_ledger.verify_chain(),
                        noise=hashlib.sha256(noise.cpu().numpy().tobytes()).hexdigest(),
                        dropped=int(eng.dpsgd.dropped.item())))
        out["dpsgd_fused"] = dict(epoch=st["epoch"], identical=len({i["digest"] for i in g}) == 1,
                                  errs=sum((i["errs"] for i in g), []), chain_ok=all(i["chain"] for i in g),
                                  noise_distinct=len({i["noise"] for i in g}) == len(g),
                                  dropped=sum(i["dropped"] for i in g), graphs=eng.graph is not None)
        torch.cuda.synchronize(); dist.barrier()
        del eng
        torch.cuda.synchronize(); dist.barrier()
    if "lora_digest" in which:
        # every rank given a different base (another genesis seed): the engine must refuse on every rank
        from bflc_demo_b200.data.synthetic import lm_corpus_like
        from bflc_demo_b200.engine.generic import GenericFedEngine
        from bflc_demo_b200.models.lora import LoRANet
        from bflc_demo_b200.models.nets import GPT
        cfg = FLConfig.for_world(world, batch_size=16, samples_per_client=64, learning_rate=2e-3, model="gpt",
                                 optimizer="adam", lora_rank=8)
        shard = lm_corpus_like(world, 64, seed=2, seq_len=128, only=rank)[0]
        refused = ""
        try:
            GenericFedEngine(cfg, LoRANet(GPT(layers=2), 8, base_seed=100 + rank), shard, rank=rank, world=world,
                             device=lr)
        except ValueError as e:
            refused = str(e)
        g = gather(dict(refused=refused))
        out["lora_digest"] = dict(refused_everywhere=all("differ" in i["refused"] for i in g),
                                  messages=[i["refused"][:80] for i in g])
        torch.cuda.synchronize(); dist.barrier()
    if rank == 0:
        print("RESULT " + json.dumps(out))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
