"""GEMM library vs cuBLAS on the shapes the model families use (VERDICT r1 item 7).

  python scripts/gemm_bench.py            -> one RESULT json line: TFLOP/s per shape and kernel

Timing: 5 warm-up calls, then 20 timed calls between CUDA events (inputs of the big shapes
exceed the 50 MB L2; the small ones are re-run over 4 rotating input sets), best and median.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from bflc_demo_b200.ops import gemm as G
from bflc_demo_b200.ops.mx8 import gemm_mx8, quantize_mx8

SHAPES = [(8192, 8192, 8192), (16384, 1024, 1024), (32768, 768, 3072), (4096, 3072, 768), (2048, 768, 768)]


def bench(fn, sets, n=20, warm=5):
    for i in range(warm):
        fn(*sets[i % len(sets)])
    torch.cuda.synchronize()
    ts = []
    for i in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(*sets[i % len(sets)])
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[0], ts[len(ts) // 2]


def main():
    out = {}
    for M, N, K in SHAPES:
        flops = 2.0 * M * N * K
        sets = [(torch.randn(M, K, device="cuda").bfloat16() * 0.1, torch.randn(N, K, device="cuda").bfloat16() * 0.1)
                for _ in range(4 if M * K * 2 < (64 << 20) else 1)]
        d = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        row = {}
        for name, fn in (("cublas", lambda a, b: torch.matmul(a, b.t(), out=d)),
                         ("ours_auto", lambda a, b: G.gemm(a, b, out=d)),
                         ("ours_pair", lambda a, b: G.gemm_2cta(a, b, out=d))):
            try:
                best, med = bench(fn, sets)
                row[name] = {"tflops_best": round(flops / best / 1e9, 1), "tflops_median": round(flops / med / 1e9, 1)}
            except Exception as e:  # noqa: BLE001
                row[name] = {"error": repr(e)[:120]}
        try:
            qs = [(quantize_mx8(a), quantize_mx8(b)) for a, b in sets]
            best, med = bench(lambda qa, qb: gemm_mx8(qa, qb, out=d), qs)
            row["ours_mxfp8"] = {"tflops_best": round(flops / best / 1e9, 1), "tflops_median": round(flops / med / 1e9, 1)}
        except Exception as e:  # noqa: BLE001
            row["ours_mxfp8"] = {"error": repr(e)[:120]}
        a, b = sets[0]
        ref = a.float() @ b.float().t() if M * N <= (1 << 26) else None
        if ref is not None:
            G.gemm_2cta(a, b, out=d)
            row["pair_rel_err"] = float(((d.float() - ref).norm() / ref.norm()).item())
        out[f"{M}x{N}x{K}"] = row
        del sets, d
        torch.cuda.empty_cache()
    print("RESULT " + json.dumps(out))


main()
