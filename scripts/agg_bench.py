"""Cost of the aggregation rule, of the server optimizer and of differential privacy inside the
consensus kernel: one-shot k_consensus per rule, and per server optimizer and DP mode on FedAvg, at the LeNet-5, ResNet-18 and BERT-base
parameter counts, K = 5 selected uploads, on one GPU.

The one-GPU replica harness (tests/test_gpu_robust_aggregation.py) emulates 6 ranks (1 committee,
5 trainers, every upload selected; the committee seat rotates, so there are always 5) and times
rank 0's one-shot consensus launch of every round with CUDA events, after warm-up rounds.  Local
HBM stands in for NVLink here: the numbers measure the rule's cost relative to FedAvg, not the
NVLink path.  Bytes that must move per launch: K * P * 4 read, fp32
global + work copies (2 * P * 4) and their bf16 shadows (2 * P * 2) written; a server optimizer
adds the global model's read (P * 4) and its state's read and write (8 B/param for momentum's m,
16 for adam / yogi's m and v).  The optimizer rows use the harness of
tests/test_gpu_server_optimizer.py.

The differential-privacy rows (FedAvg + clip, FedAvg + clip + noise, and both with the adaptive clip;
tests/test_gpu_dp.py's and tests/test_gpu_dp_adaptive.py's harnesses)
time every emulated rank's k_update_norms and rank 0's k_consensus together: the six norm launches
each reduce one slice, so together they read every upload and the global model once (K * P * 4 +
P * 4), which on a real box is spread over the GPUs; the clipping consensus kernel also reads the
global model (P * 4).  The noise adds arithmetic (one Philox call and two Box-Muller pairs per four
coordinates), no bytes.  The adaptive clip adds scalar work in thread 0 of every block (the count, one
Philox call with noise, the clip update) and one 16-byte record, no per-coordinate bytes.

    python scripts/agg_bench.py [--iters 40] [--out bench_out/agg_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

SIZES = {"lenet5": 62_006, "resnet18": 11_173_962, "bert_base": 109_483_778}
RULES = [("fedavg", 1), ("median", 1), ("trimmed_mean", 1)]
SERVER_OPTS = ["momentum", "adam", "yogi"]        # on FedAvg
DP_MODES = ["clip", "noise", "clip_adaptive", "noise_adaptive"]   # on FedAvg: clip, clip + noise, adaptive clip
K = 5


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip())


def time_rule(P: int, rule: str, trim: int, iters: int, warmup: int = 3, server_opt: str = "none",
              dp: str = "") -> dict:
    from test_gpu_dp import DpHarness
    from test_gpu_dp_adaptive import DpAdaptiveHarness
    from test_gpu_robust_aggregation import N_VAL, ReplicaHarness
    from test_gpu_server_optimizer import ServerOptHarness

    kw = dict(n_comm=1, aggregate_count=K, aggregation=rule, trim=trim)
    if dp.endswith("_adaptive"):
        noised = dp.startswith("noise")
        h = DpAdaptiveHarness(K + 1, P, clip=1.0, noise=1.0 if noised else 0.0, quantile=0.5,
                              count_noise=1.0 if noised else 0.0, **kw)
    elif dp:
        h = DpHarness(K + 1, P, clip=1.0, noise=1.0 if dp == "noise" else 0.0, **kw)
    elif server_opt == "none":
        h = ReplicaHarness(K + 1, P, **kw)
    else:
        h = ServerOptHarness(K + 1, P, server_opt=server_opt, **kw)
    rng = np.random.default_rng(0)
    ups = {t: torch.from_numpy(rng.standard_normal(P).astype(np.float32)).cuda() for t in range(K + 1)}
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for i in range(warmup + iters):
        comm = [r for r, x in enumerate(h.roles()) if x & 2]
        h.round(ups, {c: [N_VAL] * K for c in comm}, {t: 100 for t in range(K + 1)}, events=(start, stop))
        if i >= warmup:
            ts.append(start.elapsed_time(stop) * 1e3)
        errs = h.drain()        # every host ledger accepts the round (and the block ring never wraps)
        assert errs == [[]] * (K + 1), errs
    us = float(np.median(ts))
    nbytes = K * P * 4 + 2 * P * 4 + 2 * P * 2
    if server_opt != "none":
        nbytes += P * 4 + (8 if server_opt == "momentum" else 16) * P
    if dp:
        nbytes += K * P * 4 + 2 * P * 4
    name = rule if rule != "trimmed_mean" else f"trimmed_mean{trim}"
    if server_opt != "none":
        name = f"{name}+{server_opt}"
    if dp:
        name = f"{name}+dp_{dp}"
    return dict(P=P, rule=name, us_median=us,
                us_min=float(np.min(ts)), gbps=nbytes / (us * 1e-6) / 1e9, bytes=nbytes, launches=len(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "agg_bench measures the GPU kernel: no GPU found"
    out = dict(card=card(), K=K, rows=[])
    for name, P in SIZES.items():
        P8 = (P + 7) // 8 * 8
        for rule, trim, opt, dp in ([(r, t, "none", "") for r, t in RULES] + [("fedavg", 1, o, "") for o in SERVER_OPTS]
                                    + [("fedavg", 1, "none", d) for d in DP_MODES]):
            r = time_rule(P8, rule, trim, a.iters, server_opt=opt, dp=dp)
            r["model"] = name
            out["rows"].append(r)
            print(f"{name:10s} P={P8:>10d} {r['rule']:20s} {r['us_median']:9.1f} us  {r['gbps']:7.1f} GB/s",
                  flush=True)
            torch.cuda.empty_cache()
    print("RESULT " + json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
