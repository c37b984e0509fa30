"""One small federated case per process for compute-sanitizer (scripts/sanitize_gpu.sh): the
kernels with hand-rolled cross-proxy / cross-CTA synchronisation -- the persistent trainer
(bf16 and fp8, Adam, fused upload), the fp8 / bf16 validation chain, k_plan / k_consensus, the
input and blob quantisers -- at shapes small enough for racecheck.  Prints RESULT {json}."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.data.synthetic import femnist_like


def engine(dtype, optimizer, rounds=2):
    from bflc_demo_b200.engine.fused import FusedEngine
    cfg = FLConfig.for_world(1, model="mlp", hidden=256, batch_size=128, samples_per_client=256,
                             learning_rate=0.05 if optimizer == "sgd" else 1e-3, dtype=dtype,
                             optimizer=optimizer, cuda_graph=False)
    eng = FusedEngine(cfg, femnist_like(1, 256, seed=7, only=0)[0])
    for _ in range(rounds):
        eng.run_round()
    torch.cuda.synchronize()
    errs = eng.drain_blocks()
    st = eng.read_state()
    return dict(epoch=st["epoch"], loss=st["global_loss"], ledger_errs=errs, chain_ok=eng.host_ledger.verify_chain())


def conv_attn(case):
    """The round-2 kernels outside the flagship round: implicit-GEMM convolution (stride 1 and 2,
    forward + both gradients) and fused attention forward / backward, at small shapes."""
    from bflc_demo_b200.ops import nn as F
    BF = torch.bfloat16
    torch.manual_seed(0)
    if case == "conv":
        tot = 0.0
        for (n, hw, cin, cout, stride) in ((2, 16, 64, 64, 1), (2, 16, 64, 128, 2), (3, 4, 128, 64, 1)):
            x = (torch.randn(n, hw, hw, cin, device="cuda") * 0.5).to(BF).requires_grad_(True)
            w = (torch.randn(cout, 9 * cin, device="cuda") * 0.05).to(BF)
            gw = torch.zeros(cout, 9 * cin, device="cuda")
            y = F.conv2d(x, w, None, gw, None, 3, 3, stride, 1)
            y.backward(torch.ones_like(y))
            tot += float(gw.abs().sum()) + float(x.grad.float().abs().sum())
        return dict(checksum=tot)
    if case == "attn_dropout":
        # dropout instantiations: padded (lengths 1 .. 256, one sequence of length 0) and packed with
        # the same ragged lengths as attn_packed, p = 0.1
        H, S = 2, 256
        step = torch.zeros(1, device="cuda", dtype=torch.int32)
        rng = F.DropoutRNG(7, step, 3)
        q, k, v = [(torch.randn(4 * S, H * 64, device="cuda") * 0.5).to(BF).requires_grad_(True) for _ in range(3)]
        lengths = torch.tensor([256, 65, 0, 1], device="cuda", dtype=torch.int32)
        o = F.attention(q, k, v, 4, S, H, lengths=lengths, dropout_p=0.1, rng=rng, site=1)
        o.backward(torch.ones_like(o))
        total = float(o.float().abs().sum()) + float(q.grad.float().abs().sum())
        lens = [1, 63, 512, 64, 65, 10]
        cu = [0]
        for n in lens:
            cu.append(cu[-1] + n)
        qp, kp, vp = [(torch.randn(cu[-1], H * 64, device="cuda") * 0.5).to(BF).requires_grad_(True) for _ in range(3)]
        o = F.attention_packed(qp, kp, vp, torch.tensor(cu, device="cuda", dtype=torch.int32), max(lens), H,
                               dropout_p=0.1, rng=rng, site=2)
        o.backward(torch.ones_like(o))
        return dict(checksum=total + float(o.float().abs().sum()) + float(kp.grad.float().abs().sum()) +
                    float(vp.grad.float().abs().sum()))
    if case == "attn_packed":
        # packed kernels: lengths 1, 63, 64, 65 and 512, T = 715 (not a multiple of 64), the last
        # sequence ending exactly at T -- early-exit CTAs, straddling blocks, zero-filled boxes past T
        H, lens = 2, [1, 63, 512, 64, 65, 10]
        cu = [0]
        for n in lens:
            cu.append(cu[-1] + n)
        T = cu[-1]
        q, k, v = [(torch.randn(T, H * 64, device="cuda") * 0.5).to(BF).requires_grad_(True) for _ in range(3)]
        o = F.attention_packed(q, k, v, torch.tensor(cu, device="cuda", dtype=torch.int32), max(lens), H)
        o.backward(torch.ones_like(o))
        return dict(checksum=float(o.float().abs().sum()) + float(q.grad.float().abs().sum()) +
                    float(k.grad.float().abs().sum()) + float(v.grad.float().abs().sum()))
    if case == "attn_varlen":
        # tiled masked kernels: lengths 1, 0, a partial block, a full sequence (S = 192: a 128-query
        # block and a half-live one), so the K / V ring, the dQ / dK-dV barriers and the skipped
        # blocks are all exercised
        B, S, H = 4, 192, 2
        lengths = torch.tensor([1, 0, 100, S], device="cuda", dtype=torch.int32)
    else:
        B, S, H, lengths = 2, 128, 2, None
    q, k, v = [(torch.randn(B * S, H * 64, device="cuda") * 0.5).to(BF).requires_grad_(True) for _ in range(3)]
    o = F.attention(q, k, v, B, S, H, lengths=lengths)
    o.backward(torch.ones_like(o))
    return dict(checksum=float(o.float().abs().sum()) + float(q.grad.float().abs().sum()) +
                float(k.grad.float().abs().sum()) + float(v.grad.float().abs().sum()))


def main():
    case = sys.argv[1]
    if case in ("conv", "attn", "attn_varlen", "attn_packed", "attn_dropout"):
        out = dict(case=case, **conv_attn(case))
        torch.cuda.synchronize()
        print("RESULT " + json.dumps(out))
        return
    dtype, opt = case.split("_")
    out = dict(case=case, **engine(dtype, opt))
    print("RESULT " + json.dumps(out))


if __name__ == "__main__":
    main()
