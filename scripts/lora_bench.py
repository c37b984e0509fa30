"""LoRA linear, forward + backward, at BERT / GPT shapes: the tail GEMM path against the same math
composed from existing GEMMs and an add, and against today's full-fine-tuning linear.

  python scripts/lora_bench.py            -> one RESULT json line (per-shape microseconds)

(a) ``tail``: ``ops.nn.lora_linear`` -- u = s x A^T, then y = x W^T + u B^T + b as one GEMM with a
    low-rank K tail; backward v = s dz B, gB += dz^T u, gA += v^T x, dx = dz W + v A (tail GEMM).
(b) ``composed``: the same math without the tail: y = (x W^T + b) + u B^T through a second GEMM and
    an add, dx = dz W + v A through a second GEMM and an add (this script only; the library has no
    unfused LoRA path).
(c) ``full``: ``ops.nn.linear`` with its weight- and bias-gradient GEMMs (full fine-tuning; large
    plain forwards take the CTA-pair kernel).

No activation (the q / k / v / o / ff2 projections).  Each variant's forward + backward is captured
in one CUDA graph; the graph is replayed 5 times to warm up, then 30 times between CUDA events, and
the median replay is reported.  The card's name and power limit are read in the same process.
"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.autograd import Function

from bflc_demo_b200.ops import gemm as G
from bflc_demo_b200.ops import nn as F

BF = torch.bfloat16
MS = (2048, 8192)
NK = ((768, 768), (3072, 768), (768, 3072))
RANKS = (8, 16, 64)


class ComposedLoRA(Function):
    @staticmethod
    def forward(ctx, x, w, b, a, bl, ga, gbl, scale):
        y0 = G.gemm(x, w, bias=b)
        u = G.gemm(x, a, alpha=scale)
        y = F.add(y0, G.gemm(u, bl))
        ctx.save_for_backward(x, w, a, bl, u)
        ctx.ga, ctx.gbl, ctx.scale = ga, gbl, scale
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, a, bl, u = ctx.saved_tensors
        dz = dy.contiguous()
        v = G.gemm(dz, bl, b_mn=True, alpha=ctx.scale)
        F._dw(dz, u, ctx.gbl)
        F._dw(v, x, ctx.ga)
        dx = F.add(G.gemm(dz, w, b_mn=True), G.gemm(v, a, b_mn=True))
        return dx, None, None, None, None, None, None, None


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return {"name": name, "nvidia_smi": q}
    except (OSError, subprocess.SubprocessError):
        return {"name": name, "nvidia_smi": "not available"}


def time_graph(step):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    for _ in range(5):
        g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(30):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return round(ts[len(ts) // 2], 1)


def main():
    out = {"card": card(), "rows": []}
    for M in MS:
        for N, K in NK:
            gen = torch.Generator(device="cuda").manual_seed(M + N + K)
            x = (torch.randn(M, K, generator=gen, device="cuda") * 0.5).to(BF).requires_grad_(True)
            w = (torch.randn(N, K, generator=gen, device="cuda") / K ** 0.5).to(BF)
            b = torch.zeros(N, device="cuda")
            dy = torch.randn(M, N, generator=gen, device="cuda").to(BF)
            gw, gb = torch.zeros(N, K, device="cuda"), torch.zeros(N, device="cuda")

            def full():
                x.grad = None
                F.linear(x, w, b, gw, gb).backward(dy)

            row = {"M": M, "N": N, "K": K, "full_us": time_graph(full)}
            for r in RANKS:
                a = (torch.randn(r, K, generator=gen, device="cuda") / K ** 0.5).to(BF)
                bl = (torch.randn(N, r, generator=gen, device="cuda") * 0.01).to(BF)
                ga, gbl = torch.zeros(r, K, device="cuda"), torch.zeros(N, r, device="cuda")

                def tail():
                    x.grad = None
                    F.lora_linear(x, w, b, a, bl, ga, gbl, 2.0).backward(dy)

                def composed():
                    x.grad = None
                    ComposedLoRA.apply(x, w, b, a, bl, ga, gbl, 2.0).backward(dy)

                row[f"r{r}"] = {"tail_us": time_graph(tail), "composed_us": time_graph(composed)}
            out["rows"].append(row)
            print(json.dumps(row), flush=True)
    print("RESULT " + json.dumps(out))


if __name__ == "__main__":
    main()
