"""Optimizer kernels on a BERT-base-sized flat buffer: the plain Adam step, the recipe Adam step
(decoupled weight decay under the no-decay mask, linear schedule, clip coefficient read) and the
global-norm kernel that precedes it when clipping is on.

  python scripts/optim_bench.py [--iters 30] [--params N]

CUDA events around each launch, the three kernels interleaved, after a warm-up; median over
--iters (>= 20).  Achieved TB/s comes from the bytes model below (what each kernel must move per
parameter), over the median time.  The card's name, power limit and maximum SM clock are read in
the same run.  One JSON line."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch

# bytes per parameter
BYTES = {
    # read master, grad, m, v; write master, m, v, grad (cleared) in fp32 and the bf16 shadow
    "adam": 4 * 4 + 4 * 4 + 2,
    # the same plus one no-decay bit per 8 floats
    "adam_recipe": 4 * 4 + 4 * 4 + 2 + 1 / 64,
    # read grad
    "grad_norm": 4,
}


def card() -> dict:
    out = {"name": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30)
        out["power_limit"], out["max_sm_clock"] = [s.strip() for s in q.stdout.strip().split(",")]
    except (OSError, ValueError, subprocess.SubprocessError) as e:
        out["nvidia_smi_error"] = repr(e)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--params", type=int, default=0, help="flat buffer length (default: BERT-base)")
    a = ap.parse_args()
    if a.iters < 20:
        ap.error("--iters must be >= 20")
    if not torch.cuda.is_available():
        sys.exit("optim_bench needs a GPU")
    from bflc_demo_b200._native import C
    from bflc_demo_b200.models.nets import BertBase
    from bflc_demo_b200.ops.optim import OptimRecipe, RecipeStep

    spec = BertBase(2).spec
    P = a.params or spec.total
    mod = C()
    g = torch.Generator(device="cuda").manual_seed(0)
    master = torch.randn(P, device="cuda", generator=g) * 0.02
    shadow = master.to(torch.bfloat16)
    grad = torch.zeros(P, device="cuda")
    m, v = torch.zeros(P, device="cuda"), torch.zeros(P, device="cuda")
    word = torch.zeros(1, dtype=torch.int32, device="cuda")
    rs = RecipeStep(OptimRecipe(0.01, "linear", 100, 10000, 1.0), spec, 1, "cuda", n=P)
    mod.grad_norm(grad, rs.workspace, rs.norms, 0, 1.0)       # the recipe step reads its clip words

    kernels = {
        "adam": lambda: mod.optim_step(True, master, grad, shadow, m, v, 1e-5, 0.0, 0.9, 0.999, 1e-8, 1,
                                       word.data_ptr(), 0, True),
        "adam_recipe": lambda: mod.optim_recipe_step(True, master, grad, shadow, m, v, 1e-5, 0.9, 0.999, 1e-8, 1,
                                                     word.data_ptr(), 0.01, rs.mask, 1, 100, 10000, rs.workspace),
        "grad_norm": lambda: mod.grad_norm(grad, rs.workspace, rs.norms, 0, 1.0),
    }
    for _ in range(a.warmup):
        for f in kernels.values():
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in kernels}
    for _ in range(a.iters):
        for k, f in kernels.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1) * 1e3)
    res = {}
    for k, ts in times.items():
        ts = sorted(ts)
        med = ts[len(ts) // 2]
        res[k] = {"median_us": round(med, 2), "min_us": round(ts[0], 2), "max_us": round(ts[-1], 2),
                  "bytes_per_param": round(BYTES[k], 3), "tb_per_s": round(BYTES[k] * P / (med * 1e-6) / 1e12, 3)}
    line = {
        "params": P, "iters": a.iters, "card": card(), "kernels": res,
        "recipe_over_plain_adam": round(res["adam_recipe"]["median_us"] / res["adam"]["median_us"], 4),
        # bytes model only (not a measurement): what the norm pass adds to an Adam step's traffic
        "norm_traffic_share_of_adam_step": round(BYTES["grad_norm"] / BYTES["adam"], 4),
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
