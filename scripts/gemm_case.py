"""One GEMM bring-up case per process (a device trap poisons the context). Prints a JSON line."""
import os as _os, sys as _sys
_sys.path.insert(0, _os.path.dirname(_os.path.dirname(_os.path.abspath(__file__))))
import json, sys, time
import torch
from bflc_demo_b200.ops import gemm as G
from bflc_demo_b200._native import C

def rel_err(x, ref):
    return ((x.float() - ref.float()).norm() / (ref.float().norm() + 1e-12)).item()

def main():
    case = sys.argv[1]
    torch.manual_seed(0)
    dev = "cuda"
    out = {"case": case}
    def mk(*shape):
        # rows must start on 16-byte boundaries for TMA: pad the contiguous dim to x8, slice
        c = shape[-1]; cp = (c + 7) // 8 * 8
        t = (torch.randn(*shape[:-1], cp, device=dev) * 0.5).to(torch.bfloat16)
        return t[..., :c] if cp != c else t
    if case.startswith("kk"):           # kk_M_N_K
        _, M, N, K = case.split("_"); M, N, K = int(M), int(N), int(K)
        a, b = mk(M, K), mk(N, K)
        d = G.gemm(a, b, out_dtype=torch.float32)
        ref = a.float() @ b.float().t()
        out["err"] = rel_err(d, ref)
    elif case.startswith("kmn"):        # A K-major, B MN-major [K,N]; optional lbo/sbo override
        parts = case.split("_"); M, N, K = map(int, parts[1:4])
        dbg = (0, 0, int(parts[4]), int(parts[5])) if len(parts) > 4 else (0, 0, 0, 0)
        a, b = mk(M, K), mk(K, N)
        d = G.gemm(a, b, b_mn=True, out_dtype=torch.float32, dbg=dbg)
        out["err"] = rel_err(d, a.float() @ b.float())
    elif case.startswith("mnmn"):       # A [K,M], B [K,N]
        parts = case.split("_"); M, N, K = map(int, parts[1:4])
        dbg = (int(parts[4]), int(parts[5]), int(parts[4]), int(parts[5])) if len(parts) > 4 else (0, 0, 0, 0)
        a, b = mk(K, M), mk(K, N)
        d = G.gemm(a, b, a_mn=True, b_mn=True, out_dtype=torch.float32, dbg=dbg)
        out["err"] = rel_err(d, a.float().t() @ b.float())
    elif case.startswith("fp8"):
        _, M, N, K = case.split("_"); M, N, K = int(M), int(N), int(K)
        a = (torch.randn(M, K, device=dev) * 0.5).to(torch.float8_e4m3fn)
        b = (torch.randn(N, K, device=dev) * 0.5).to(torch.float8_e4m3fn)
        d = G.gemm(a, b, out_dtype=torch.float32)
        out["err"] = rel_err(d, a.float() @ b.float().t())
    elif case == "epi":
        M, N, K = 300, 200, 784
        a, b = mk(M, K), mk(N, K)
        bias = torch.randn(N, device=dev)
        colsum = torch.zeros(N, device=dev)
        d = G.gemm(a, b, bias=bias, act=G.ACT_RELU, colsum=colsum)
        ref = torch.relu(a.float() @ b.float().t() + bias)
        out["err_relu"] = rel_err(d, ref)
        out["err_colsum"] = rel_err(colsum, ref.sum(0))
        d2 = G.gemm(a, b, split_k=4)
        out["err_splitk"] = rel_err(d2, a.float() @ b.float().t())
        mask = mk(M, N)
        d3 = G.gemm(a, b, aux_in=mask, act_bwd=1, out_dtype=torch.float32)
        out["err_relubwd"] = rel_err(d3, (a.float() @ b.float().t()) * (mask.float() > 0))
        # batched
        ab, bb = mk(3, 130, 64), mk(3, 70, 64)
        d4 = G.gemm(ab, bb, out_dtype=torch.float32)
        out["err_batched"] = rel_err(d4, torch.bmm(ab.float(), bb.float().transpose(1, 2)))
    elif case == "xent":
        M, N, K = 500, 62, 256
        a, b = mk(M, K), mk(N, K)
        bias = torch.randn(N, device=dev) * 0.1
        labels = torch.randint(0, N, (M,), device=dev, dtype=torch.int32)
        dl = torch.full((M, 64), 7.0, device=dev, dtype=torch.bfloat16)
        loss = torch.zeros(1, device=dev); corr = torch.zeros(1, device=dev, dtype=torch.int32)
        colsum = torch.zeros(N, device=dev)
        G.gemm_xent(a, b, labels, n_classes=N, bias=bias, dlogits=dl, grad_scale=1.0 / M,
                    loss_sum=loss, correct=corr, colsum=colsum)
        logits = a.float() @ b.float().t() + bias
        ref_loss = torch.nn.functional.cross_entropy(logits, labels.long(), reduction="sum")
        p = torch.softmax(logits, 1); p[torch.arange(M), labels.long()] -= 1; p /= M
        out["err_loss"] = abs(loss.item() - ref_loss.item()) / abs(ref_loss.item())
        out["err_dlogits"] = rel_err(dl[:, :N], p)
        out["pad_zero"] = bool((dl[:, N:] == 0).all().item())
        out["correct"] = [int(corr.item()), int((logits.argmax(1) == labels).sum().item())]
        out["err_colsum"] = rel_err(colsum, p.sum(0))
        corr2 = torch.zeros(2, device=dev, dtype=torch.int32)
        G.gemm_argmax_acc(a, b, labels, corr2, n_classes=N, bias=bias)
        out["argmax_correct"] = int(corr2[0].item())
    elif case == "perf":
        res = {}
        for (M, N, K) in [(8192, 8192, 8192), (4096, 4096, 4096), (16384, 256, 784), (16384, 1024, 784)]:
            a, b = mk(M, K), mk(N, K)
            o = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            for _ in range(3): G.gemm(a, b, out=o)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10): G.gemm(a, b, out=o)
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 10
            for _ in range(3): torch.matmul(a, b.t(), out=o)
            e0.record()
            for _ in range(10): torch.matmul(a, b.t(), out=o)
            e1.record(); torch.cuda.synchronize()
            ms_t = e0.elapsed_time(e1) / 10
            res[f"{M}x{N}x{K}"] = {"ours_ms": ms, "ours_tflops": 2 * M * N * K / ms / 1e9,
                                   "cublas_ms": ms_t, "cublas_tflops": 2 * M * N * K / ms_t / 1e9}
        out["perf"] = res
    elif case == "perf_small":
        a, b = mk(512, 784), mk(256, 784)
        bias = torch.randn(256, device=dev)
        o = torch.empty(512, 256, device=dev, dtype=torch.bfloat16)
        for _ in range(36): G.gemm(a, b, out=o, bias=bias, act=G.ACT_RELU)
    elif case == "perf_big":
        a, b = mk(8192, 8192), mk(8192, 8192)
        o = torch.empty(8192, 8192, device=dev, dtype=torch.bfloat16)
        for _ in range(5): G.gemm(a, b, out=o)
    elif case == "perf2":
        res = {}
        for (M, N, K) in [(8192, 8192, 8192), (4096, 4096, 4096), (16384, 1024, 784), (32768, 768, 3072)]:
            a, b = mk(M, K), mk(N, K)
            o = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            def t(fn):
                for _ in range(3): fn()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(10): fn()
                e1.record(); torch.cuda.synchronize()
                return e0.elapsed_time(e1) / 10
            m1 = t(lambda: G.gemm(a, b, out=o))
            m3 = t(lambda: torch.matmul(a, b.t(), out=o))
            f = 2 * M * N * K / 1e9
            res[f"{M}x{N}x{K}"] = {"ours_tflops": f / m1, "cublas_tflops": f / m3}
        out["perf2"] = res
    elif case == "perf3":      # block-scaled fp8 vs per-tensor fp8 vs bf16 vs cuBLAS bf16
        from bflc_demo_b200.ops.mx8 import gemm_mx8, quantize_mx8
        res = {}
        for (M, N, K) in [(8192, 8192, 8192), (4096, 4096, 4096), (16384, 1024, 1024), (4096, 256, 784)]:
            a, b = mk(M, K), mk(N, K)
            qa, qb = quantize_mx8(a), quantize_mx8(b)
            fa, fb = a.to(torch.float8_e4m3fn), b.to(torch.float8_e4m3fn)
            o = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            def t(fn):
                for _ in range(3): fn()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(10): fn()
                e1.record(); torch.cuda.synchronize()
                return e0.elapsed_time(e1) / 10
            f = 2 * M * N * K / 1e9
            res[f"{M}x{N}x{K}"] = {
                "mx8_tflops": f / t(lambda: gemm_mx8(qa, qb, out=o)),
                "fp8_pertensor_tflops": f / t(lambda: G.gemm(fa, fb, out=o)),
                "bf16_tflops": f / t(lambda: G.gemm(a, b, out=o)),
                "cublas_bf16_tflops": f / t(lambda: torch.matmul(a, b.t(), out=o)),
                "quantize_a_us": 1e3 * t(lambda: quantize_mx8(a, out=qa)),
                "mx8_err_vs_bf16": rel_err(gemm_mx8(qa, qb, out_dtype=torch.float32), a.float() @ b.float().t())}
        out["perf3"] = res
    elif case.startswith("ncu_"):   # a few launches of one kernel for a profiler capture
        from bflc_demo_b200.ops.mx8 import gemm_mx8, quantize_mx8
        a, b = mk(8192, 8192), mk(8192, 8192)
        o = torch.empty(8192, 8192, device=dev, dtype=torch.bfloat16)
        if case == "ncu_1cta":
            for _ in range(3): G.gemm(a, b, out=o)
        elif case == "ncu_mx8":
            qa, qb = quantize_mx8(a), quantize_mx8(b)
            for _ in range(3): gemm_mx8(qa, qb, out=o)
    elif case == "elem":
        n = 100003
        x = torch.randn(n, device=dev)
        y = torch.empty(n, device=dev, dtype=torch.bfloat16)
        C().cast_f32_to_bf16(x, y)
        out["cast"] = rel_err(y, x.bfloat16())
        u = torch.randint(0, 255, (n,), device=dev, dtype=torch.uint8)
        C().cast_u8_to_bf16(u, y, 1 / 255.)
        out["u8"] = rel_err(y, (u.float() / 255).bfloat16())
        # optimizers
        for adam in (False, True):
            w = torch.randn(n + 1, device=dev); g = torch.randn(n + 1, device=dev)
            w0, g0 = w.clone(), g.clone()
            sh = torch.empty(n + 1, device=dev, dtype=torch.bfloat16)
            m = torch.zeros_like(w); v = torch.zeros_like(w)
            C().optim_step(adam, w, g, sh, m, v, 1e-2, 0.0, 0.9, 0.999, 1e-8, 1, 0, 0, True)
            if adam:
                ref = w0 - 1e-2 * g0 / (g0.abs() + 1e-8)
            else:
                ref = w0 - 1e-2 * g0
            out["adam" if adam else "sgd"] = rel_err(w, ref)
            out["shadow_%d" % adam] = rel_err(sh, ref.bfloat16())
            out["zeroed_%d" % adam] = bool((g == 0).all().item())
    torch.cuda.synchronize()
    out["ok"] = True
    print("RESULT " + json.dumps(out))

if __name__ == "__main__":
    main()
