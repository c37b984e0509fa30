"""Attention forward + backward at BERT-base head shapes (H = 12, D = 64), graph-replayed, CUDA
events, L2 flushed between iterations.  Sequence lengths S = 128 / 256 / 512, each once at full
length and once with per-sequence lengths uniform in [S/4, S] (right padding).  Arms:

  tiled     the tiled online-softmax kernels (csrc/kernels/attn_sm100.cu), given a lengths tensor
  packed    the same kernels in packed mode: the real rows only, concatenated, with cu_seqlens
  whole     the one-CTA-per-head S = 128 kernel (unmasked S = 128 only)
  unfused   batched GEMMs + softmax kernel + head transposes (mask-free, so full length only)
  sdpa      torch scaled_dot_product_attention with the boolean key mask, as a reference

``--dropout``: instead, attention-probability dropout p = 0.1 against p = 0 on the tiled and packed
arms, at full and variable length (tiled_drop_us / packed_drop_us, and their ratios to p = 0).

``--causal``: instead, the causal kernels (query i attends to keys j <= i, the key blocks above the
diagonal skipped) against the same tiled kernels unmasked and sdpa with is_causal, full length only
(causal_us, tiled_us, sdpa_causal_us, causal_speedup = tiled_us / causal_us).  TFLOP/s there counts
the S (S + 1) / 2 visible (query, key) pairs.

TFLOP/s counts the valid key positions only: 4 * S * len_b * D per (sequence, head) forward, times
3.5 for forward + backward (2 GEMMs forward, 5 backward), so a masked run that skips the padded
keys is credited with the work it had to do, not with the padded work."""
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


def case(B, S, varlen, H=12, D=64):
    gen = torch.Generator().manual_seed(S + B)
    if varlen:
        lens = torch.randint(S // 4, S + 1, (B,), generator=gen, dtype=torch.int32)
    else:
        lens = torch.full((B,), S, dtype=torch.int32)
    lengths = lens.cuda()
    q, k, v = [(torch.randn(B * S, H * D, device="cuda") * 0.5).to(BF).requires_grad_(True) for _ in range(3)]
    do = torch.randn(B * S, H * D, device="cuda").to(BF)

    step = torch.zeros(1, device="cuda", dtype=torch.int32)
    rng = F.DropoutRNG(1234, step)

    def ours(**kw):
        def f():
            q.grad = k.grad = v.grad = None
            o = F.attention(q, k, v, B, S, H, **kw)
            o.backward(do)
        return f
    q4, k4, v4 = [t.detach().view(B, S, H, D).transpose(1, 2).contiguous().requires_grad_(True) for t in (q, k, v)]
    do4 = do.view(B, S, H, D).transpose(1, 2).contiguous()
    mask = (torch.arange(S, device="cuda")[None, :] < lengths[:, None].long()).view(B, 1, 1, S)

    def sdpa():
        q4.grad = k4.grad = v4.grad = None
        o = TF.scaled_dot_product_attention(q4, k4, v4, attn_mask=mask)
        o.backward(do4)
    real = (torch.arange(S)[None, :] < lens[:, None]).view(-1).cuda()
    qp, kp, vp = [t.detach()[real].requires_grad_(True) for t in (q, k, v)]
    dop = do[real]
    cu = torch.cat([torch.zeros(1, dtype=torch.int32), torch.cumsum(lens, 0, dtype=torch.int32)]).cuda()

    def packed(p=0.0):
        def f():
            qp.grad = kp.grad = vp.grad = None
            o = F.attention_packed(qp, kp, vp, cu, int(lens.max()), H, dropout_p=p, rng=rng, site=1)
            o.backward(dop)
        return f
    if CAUSAL:
        pairs = 3.5 * 4 * H * D * B * S * (S + 1) / 2

        def sdpa_causal():
            q4.grad = k4.grad = v4.grad = None
            TF.scaled_dot_product_attention(q4, k4, v4, is_causal=True).backward(do4)
        r = dict(batch=B, seq=S, causal_us=timed(ours(causal=True)), tiled_us=timed(ours(lengths=lengths)),
                 sdpa_causal_us=timed(sdpa_causal))
        r["causal_speedup"] = round(r["tiled_us"] / r["causal_us"], 3)
        r["causal_tflops"] = round(pairs / r["causal_us"] / 1e6, 1)
        return r
    if DROPOUT:
        r = dict(batch=B, seq=S, varlen=varlen, tiled_us=timed(ours(lengths=lengths)),
                 tiled_drop_us=timed(ours(lengths=lengths, dropout_p=0.1, rng=rng, site=1)),
                 packed_us=timed(packed()), packed_drop_us=timed(packed(0.1)))
        r["tiled_drop_ratio"] = round(r["tiled_drop_us"] / r["tiled_us"], 3)
        r["packed_drop_ratio"] = round(r["packed_drop_us"] / r["packed_us"], 3)
        return r
    flops = 3.5 * 4 * H * S * D * float(lens.sum())
    r = dict(batch=B, seq=S, varlen=varlen, valid_key_fraction=round(float(lens.sum()) / (B * S), 3),
             tiled_us=timed(ours(lengths=lengths)), packed_us=timed(packed()))
    if S == 128 and not varlen:
        r["whole_us"] = timed(ours())
    if not varlen:
        r["unfused_us"] = timed(ours(fused=False))
    r["sdpa_us"] = timed(sdpa)
    for arm in ("tiled", "packed", "whole", "unfused", "sdpa"):
        if f"{arm}_us" in r:
            r[f"{arm}_tflops"] = round(flops / r[f"{arm}_us"] / 1e6, 1)
    return r


DROPOUT = "--dropout" in sys.argv[1:]
CAUSAL = "--causal" in sys.argv[1:]
out = []
for S in (128, 256, 512):
    for B in (16, 64):
        for varlen in ((False,) if CAUSAL else (False, True)):
            r = case(B, S, varlen)
            out.append(r); print(json.dumps(r), flush=True)
            torch.cuda.empty_cache()
print("ATTN_BENCH " + json.dumps(out))
