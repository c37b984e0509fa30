"""Tiled attention with per-sequence lengths (attn_sm100.cu): against fp32 SDPA with a boolean key
mask, masked positions inert, deterministic and graph-capturable backward, and padded BERT end to
end (padding invariance, exactly-zero gradients for padding, two captured engine rounds)."""
import math

import pytest
import torch
import torch.nn.functional as TF

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
D = 64


def rel(x, ref):
    return ((x.float() - ref.float()).norm() / (ref.float().norm() + 1e-12)).item()


@pytest.fixture(scope="module")
def F():
    from bflc_demo_b200.ops import nn
    return nn


def _qkv(B, S, H, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [(torch.randn(B * S, H * D, device="cuda", generator=g) * 0.7).to(BF).requires_grad_(True)
            for _ in range(3)]


def _run(F, q, k, v, do, B, S, H, lengths):
    for t in (q, k, v):
        t.grad = None
    o = F.attention(q, k, v, B, S, H, lengths=lengths)
    o.backward(do)
    return o.detach(), q.grad.clone(), k.grad.clone(), v.grad.clone()


def _sdpa_ref(q, k, v, do, B, S, H, lengths):
    def heads(t):
        return t.view(B, S, H, D).permute(0, 2, 1, 3)
    qr, kr, vr = (t.detach().float().requires_grad_(True) for t in (q, k, v))
    mask = None
    if lengths is not None:
        mask = (torch.arange(S, device="cuda")[None, :] < lengths[:, None].long()).view(B, 1, 1, S)
    o = TF.scaled_dot_product_attention(heads(qr), heads(kr), heads(vr), attn_mask=mask)
    o = o.permute(0, 2, 1, 3).reshape(B * S, H * D)
    o.backward(do.float())
    return o, qr.grad, kr.grad, vr.grad


@pytest.mark.parametrize("S", [64, 128, 256, 512])
def test_masked_matches_sdpa(F, S):
    torch.manual_seed(S)
    lens = [1, 63, 64, 65, S, int(torch.randint(1, S + 1, (1,))), int(torch.randint(1, S + 1, (1,)))]
    B, H = len(lens), 2
    lengths = torch.tensor(lens, device="cuda", dtype=torch.int32)   # 65 > S = 64 clamps to S
    q, k, v = _qkv(B, S, H, S)
    do = torch.randn(B * S, H * D, device="cuda").to(BF)
    o, dq, dk, dv = _run(F, q, k, v, do, B, S, H, lengths)
    ro, rq, rk, rv = _sdpa_ref(q, k, v, do, B, S, H, lengths.clamp(max=S))
    assert rel(o, ro) < 2e-2
    assert rel(dq, rq) < 5e-2 and rel(dk, rk) < 5e-2 and rel(dv, rv) < 5e-2


@pytest.mark.parametrize("S", [192, 256, 512])
def test_unmasked_fused_route_matches_sdpa(F, S):
    B, H = 3, 4
    q, k, v = _qkv(B, S, H, 10 + S)
    do = torch.randn(B * S, H * D, device="cuda").to(BF)
    o, dq, dk, dv = _run(F, q, k, v, do, B, S, H, None)
    ro, rq, rk, rv = _sdpa_ref(q, k, v, do, B, S, H, None)
    assert rel(o, ro) < 2e-2
    assert rel(dq, rq) < 5e-2 and rel(dk, rk) < 5e-2 and rel(dv, rv) < 5e-2


def test_lengths_outside_fused_shapes_raise(F):
    q, k, v = _qkv(1, 96, 1, 0)
    lengths = torch.tensor([50], device="cuda", dtype=torch.int32)
    with pytest.raises(ValueError):
        F.attention(q, k, v, 1, 96, 1, lengths=lengths)
    q, k, v = _qkv(1, 128, 1, 0)
    with pytest.raises(ValueError):
        F.attention(q, k, v, 1, 128, 1, fused=False, lengths=torch.tensor([50], device="cuda", dtype=torch.int32))


def test_masked_positions_are_inert(F):
    B, S, H = 4, 256, 2
    lens = [1, 100, 192, 0]
    lengths = torch.tensor(lens, device="cuda", dtype=torch.int32)
    q, k, v = _qkv(B, S, H, 3)
    do = torch.randn(B * S, H * D, device="cuda").to(BF)
    o, dq, dk, dv = _run(F, q, k, v, do, B, S, H, lengths)
    pad = torch.zeros(B, S, dtype=torch.bool, device="cuda")
    for b, n in enumerate(lens):
        pad[b, max(n, 0):] = True
    pad = pad.view(B * S)
    # other finite values in the masked K / V rows leave the output bit for bit unchanged
    k2, v2 = k.detach().clone(), v.detach().clone()
    k2[pad] = (torch.randn(int(pad.sum()), H * D, device="cuda") * 3).to(BF)
    v2[pad] = (torch.randn(int(pad.sum()), H * D, device="cuda") * 3).to(BF)
    k2.requires_grad_(True); v2.requires_grad_(True)
    o2, dq2, _, _ = _run(F, q, k2, v2, do, B, S, H, lengths)
    assert torch.equal(o, o2) and torch.equal(dq, dq2)
    assert torch.count_nonzero(dk[pad]) == 0 and torch.count_nonzero(dv[pad]) == 0
    # length 0: zero output and gradients, nothing non-finite
    z = slice(3 * S, 4 * S)
    for t in (o, dq, dk, dv):
        assert torch.isfinite(t.float()).all()
        assert torch.count_nonzero(t[z]) == 0


def test_backward_deterministic_and_graph_replay_bit_identical(F):
    B, S, H = 3, 384, 4
    lengths = torch.tensor([384, 200, 65], device="cuda", dtype=torch.int32)
    q, k, v = _qkv(B, S, H, 7)
    do = torch.randn(B * S, H * D, device="cuda").to(BF)
    first = _run(F, q, k, v, do, B, S, H, lengths)
    second = _run(F, q, k, v, do, B, S, H, lengths)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    g = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        _run(F, q, k, v, do, B, S, H, lengths)          # warm-up on the capture stream
        with torch.cuda.graph(g, stream=st):
            for t in (q, k, v):
                t.grad = None
            o = F.attention(q, k, v, B, S, H, lengths=lengths)
            o.backward(do)
    torch.cuda.current_stream().wait_stream(st)
    for t in (q, k, v):
        t.grad.zero_()
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(first, (o, q.grad, k.grad, v.grad)):
        assert torch.equal(a, b)


def _bert(pad_id=0, layers=2):
    from bflc_demo_b200.models.nets import BertBase
    net = BertBase(2, layers=layers, pad_id=pad_id)
    master = torch.empty(net.spec.total)
    net.init_(master, seed=1)
    master = master.cuda()
    shadow = master.to(BF)
    grad = torch.zeros_like(master)
    return net, net.bind(master, shadow, grad), grad


def _padded(tokens, S):
    ids = torch.zeros(len(tokens), S, dtype=torch.int32, device="cuda")
    for i, t in enumerate(tokens):
        ids[i, :len(t)] = t
    return ids


def test_bert_padding_invariance_and_zero_pad_gradients():
    torch.manual_seed(11)
    lens = [128, 100, 37, 5]
    tokens = [torch.randint(1, 30522, (n,), dtype=torch.int32, device="cuda") for n in lens]
    net, b, grad = _bert()
    with torch.no_grad():
        h128 = net.features(b, _padded(tokens, 128), False)
        h256 = net.features(b, _padded(tokens, 256), False)
    assert rel(h256, h128) < 2e-2
    y = torch.tensor([0, 1, 1, 0], device="cuda", dtype=torch.int32)
    loss = net.loss(b, _padded(tokens, 256), y)
    loss.backward()
    G = net.spec.views(grad)
    assert float(G["emb.word"].abs().sum()) > 0
    assert torch.count_nonzero(G["emb.word"][0]) == 0                 # the pad token
    assert torch.count_nonzero(G["emb.pos"][max(lens):]) == 0         # positions only padding reaches
    assert torch.count_nonzero(G["emb.pos"][:max(lens)]) > 0


def test_padded_bert_generic_engine_two_captured_rounds():
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import tokens_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import BertBase
    cfg = FLConfig.for_world(1, model="bert", batch_size=8, samples_per_client=16, learning_rate=0.002)
    shard = tokens_like(1, 16, seed=3, seq_len=256, min_len=64)[0]
    eng = GenericFedEngine(cfg, BertBase(shard.n_classes, layers=2, pad_id=0), shard, rank=0, world=1, device=0)
    eng.capture()
    assert eng.graph_train is not None and not eng.capture_error
    for _ in range(2):
        eng.run_round()
    st = eng.read_state()
    assert math.isfinite(st["global_loss"])
    assert eng.drain_blocks() == [] and eng.host_ledger.verify_chain()
