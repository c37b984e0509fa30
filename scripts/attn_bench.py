"""Fused seq-128 attention (csrc/kernels/attn_sm100.cu) vs the unfused path (batched wgmma GEMMs +
softmax kernel) vs torch SDPA (flash), forward + backward, BERT-base shapes, graph-replayed,
CUDA events, L2 flushed between iterations."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as TF
from bflc_demo_b200.ops import nn as F
BF = torch.bfloat16


def timed(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph(); st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        fn()
        with torch.cuda.graph(g, stream=st):
            fn()
    torch.cuda.synchronize()
    flush = torch.empty(256 << 20, device="cuda", dtype=torch.uint8)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        flush.zero_(); a.record(); g.replay(); b.record()
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) for a, b in ev)
    return round(ts[len(ts) // 2] * 1e3, 1)


out = []
for B in (16, 64):
    S, H, D = 128, 12, 64
    q, k, v = [(torch.randn(B * S, H * D, device="cuda") * 0.5).to(BF).requires_grad_(True) for _ in range(3)]
    do = torch.randn(B * S, H * D, device="cuda").to(BF)

    def ours(fused):
        def f():
            q.grad = k.grad = v.grad = None
            o = F.attention(q, k, v, B, S, H, fused=fused)
            o.backward(do)
        return f
    q4, k4, v4 = [t.detach().view(B, S, H, D).transpose(1, 2).contiguous().requires_grad_(True) for t in (q, k, v)]
    do4 = do.view(B, S, H, D).transpose(1, 2).contiguous()

    def sdpa():
        q4.grad = k4.grad = v4.grad = None
        o = TF.scaled_dot_product_attention(q4, k4, v4)
        o.backward(do4)
    flops = 3.5 * 4 * B * H * S * S * D      # fwd 2 GEMMs + bwd 5 GEMMs
    r = dict(batch=B, fused_us=timed(ours(True)), unfused_us=timed(ours(False)), sdpa_us=timed(sdpa))
    r["fused_tflops"] = round(flops / r["fused_us"] / 1e6, 1)
    out.append(r); print(json.dumps(r), flush=True)
print("ATTN_BENCH " + json.dumps(out))
