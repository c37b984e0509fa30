"""Packed variable-length attention (attn_sm100.cu, packed mode) and packed BERT: against fp32 SDPA
per sequence, writes confined to the sequences' rows, bit-identical to the padded masked kernels on
the same tokens, deterministic and graph-capturable, and packed BERT against padded BERT, alone and
through two captured engine rounds."""
import math

import pytest
import torch
import torch.nn.functional as TF

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
D = 64
RAGGED = [1, 63, 64, 65, 127, 128, 129, 300, 511, 512]


def rel(x, ref):
    return ((x.float() - ref.float()).norm() / (ref.float().norm() + 1e-12)).item()


@pytest.fixture(scope="module")
def F():
    from bflc_demo_b200.ops import nn
    return nn


def _cu(lens):
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    return cu


def _packed_qkv(T, H, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [(torch.randn(T, H * D, device="cuda", generator=g) * 0.7).to(BF).requires_grad_(True)
            for _ in range(3)]


def _run_packed(F, q, k, v, do, cu, max_len, H):
    for t in (q, k, v):
        t.grad = None
    o = F.attention_packed(q, k, v, cu, max_len, H)
    o.backward(do)
    return o.detach(), q.grad.clone(), k.grad.clone(), v.grad.clone()


@pytest.mark.parametrize("H", [1, 3])
def test_packed_matches_sdpa_per_sequence(F, H):
    lens = RAGGED
    cu = _cu(lens)
    T = cu[-1]
    q, k, v = _packed_qkv(T, H, 100 + H)
    do = torch.randn(T, H * D, device="cuda").to(BF)
    cu_d = torch.tensor(cu, device="cuda", dtype=torch.int32)
    o, dq, dk, dv = _run_packed(F, q, k, v, do, cu_d, max(lens), H)
    refs = [torch.empty(T, H * D, device="cuda") for _ in range(4)]
    for b, n in enumerate(lens):
        rows = slice(cu[b], cu[b + 1])

        def heads(t):
            return t[rows].view(1, n, H, D).permute(0, 2, 1, 3)
        qr, kr, vr = (t.detach().float().requires_grad_(True) for t in (q, k, v))
        ob = TF.scaled_dot_product_attention(heads(qr), heads(kr), heads(vr))
        ob = ob.permute(0, 2, 1, 3).reshape(n, H * D)
        ob.backward(do[rows].float())
        refs[0][rows] = ob.detach()
        for r, t in zip(refs[1:], (qr, kr, vr)):
            r[rows] = t.grad[rows]
    assert rel(o, refs[0]) < 2e-2
    assert rel(dq, refs[1]) < 5e-2 and rel(dk, refs[2]) < 5e-2 and rel(dv, refs[3]) < 5e-2


def test_packed_op_rejects_bad_shapes(F):
    q, k, v = _packed_qkv(100, 2, 0)
    cu = torch.tensor([0, 100], device="cuda", dtype=torch.int32)
    with pytest.raises(ValueError):
        F.attention_packed(q, k, v, cu, 100, 4)          # head dim 32
    with pytest.raises(ValueError):
        F.attention_packed(q, k, v, cu, 513, 2)
    with pytest.raises(ValueError):
        F.attention_packed(q, k, v, cu, 0, 2)


def test_packed_writes_only_sequence_rows():
    """Outputs start as NaN inside [0, T) and as a sentinel past T in a larger allocation: after
    forward and backward no NaN is left in [0, T), and every sentinel row is bit-unchanged."""
    from bflc_demo_b200._native import C
    lens = [65, 1, 200, 37, 64, 129]              # T = 496: not a multiple of 64, ends exactly at T
    cu = _cu(lens)
    T, H, extra = cu[-1], 2, 80
    cu_d = torch.tensor(cu, device="cuda", dtype=torch.int32)
    S_pad = (max(lens) + 63) // 64 * 64
    g = torch.Generator(device="cuda").manual_seed(4)
    sentinel = torch.full((extra, H * D), 3.25, device="cuda", dtype=BF)
    bufs = {}
    for name in ("q", "k", "v", "do"):
        t = torch.empty(T + extra, H * D, device="cuda", dtype=BF)
        t[:T] = (torch.randn(T, H * D, device="cuda", generator=g) * 0.7).to(BF)
        t[T:] = sentinel
        bufs[name] = t
    for name in ("o", "dq", "dk", "dv"):
        t = torch.full((T + extra, H * D), float("nan"), device="cuda", dtype=BF)
        t[T:] = sentinel
        bufs[name] = t
    lse = torch.empty(len(lens) * H * S_pad, device="cuda")
    delta = torch.empty_like(lse)
    v_ = {n: t[:T] for n, t in bufs.items()}
    C().attention_packed_fwd(v_["q"], v_["k"], v_["v"], v_["o"], lse, cu_d, max(lens), H, 0.125)
    C().attention_packed_bwd(v_["q"], v_["k"], v_["v"], v_["o"], v_["do"], lse, v_["dq"], v_["dk"], v_["dv"],
                             delta, cu_d, max(lens), H, 0.125)
    torch.cuda.synchronize()
    for name, t in bufs.items():
        assert not torch.isnan(t[:T].float()).any(), name
        assert torch.equal(t[T:].view(torch.int16), sentinel.view(torch.int16)), name


def test_packed_bit_identical_to_padded(F):
    """The same tokens through the padded masked kernels: masked columns contribute exact zeros
    in the same summation order, so o and dq match bit for bit, and dk / dv too when dO is zero on
    the padded rows (the padded kernels still compute padded query rows)."""
    S, H = 256, 2
    lens = [1, 63, 64, 65, 129, 256, 200]
    B, cu = len(lens), _cu(lens)
    T = cu[-1]
    g = torch.Generator(device="cuda").manual_seed(9)
    padded = [(torch.randn(B * S, H * D, device="cuda", generator=g) * 0.7).to(BF) for _ in range(3)]
    do_p = torch.randn(B * S, H * D, device="cuda", generator=g).to(BF)
    real = torch.zeros(B * S, dtype=torch.bool, device="cuda")
    for b, n in enumerate(lens):
        real[b * S:b * S + n] = True
    do_p[~real] = 0
    packed = [t[real].clone().requires_grad_(True) for t in padded]
    padded = [t.requires_grad_(True) for t in padded]
    lengths = torch.tensor(lens, device="cuda", dtype=torch.int32)
    for t in padded:
        t.grad = None
    o_p = F.attention(*padded, B, S, H, lengths=lengths)
    o_p.backward(do_p)
    ref = [o_p.detach()[real]] + [t.grad[real] for t in padded]
    got = _run_packed(F, *packed, do_p[real], torch.tensor(cu, device="cuda", dtype=torch.int32), max(lens), H)
    for name, a, b in zip(("o", "dq", "dk", "dv"), got, ref):
        assert torch.equal(a, b), f"{name}: max |d| = {(a.float() - b.float()).abs().max().item()}"


def test_packed_deterministic_and_graph_replay_bit_identical(F):
    lens = [384, 200, 65, 1, 129]
    H = 4
    cu = torch.tensor(_cu(lens), device="cuda", dtype=torch.int32)
    T = sum(lens)
    q, k, v = _packed_qkv(T, H, 7)
    do = torch.randn(T, H * D, device="cuda").to(BF)
    first = _run_packed(F, q, k, v, do, cu, max(lens), H)
    second = _run_packed(F, q, k, v, do, cu, max(lens), H)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    g = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        _run_packed(F, q, k, v, do, cu, max(lens), H)          # warm-up on the capture stream
        with torch.cuda.graph(g, stream=st):
            for t in (q, k, v):
                t.grad = None
            o = F.attention_packed(q, k, v, cu, max(lens), H)
            o.backward(do)
    torch.cuda.current_stream().wait_stream(st)
    for t in (q, k, v):
        t.grad.zero_()
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(first, (o, q.grad, k.grad, v.grad)):
        assert torch.equal(a, b)


def _bert(packed, layers=2):
    from bflc_demo_b200.models.nets import BertBase
    net = BertBase(2, layers=layers, pad_id=0, packed=packed)
    master = torch.empty(net.spec.total)
    net.init_(master, seed=1)
    master = master.cuda()
    shadow = master.to(BF)
    grad = torch.zeros_like(master)
    return net, net.bind(master, shadow, grad), grad


def test_bert_packed_matches_padded():
    torch.manual_seed(11)
    lens, S = [128, 100, 37, 5], 256
    ids = torch.zeros(len(lens), S, dtype=torch.int64, device="cuda")
    for i, n in enumerate(lens):
        ids[i, :n] = torch.randint(1, 30522, (n,), device="cuda")
    y = torch.tensor([0, 1, 1, 0], device="cuda", dtype=torch.int32)
    out = {}
    for packed in (False, True):
        net, b, grad = _bert(packed)
        x = net.preprocess(ids)
        with torch.no_grad():
            h = net.features(b, x, False)
        loss = net.loss(b, x, y)
        loss.backward()
        torch.cuda.synchronize()
        out[packed] = (h.float(), float(loss.detach()), grad.clone(), net.spec.views(grad))
    (hp, lp, gp, _), (hk, lk, gk, G) = out[False], out[True]
    assert rel(hk, hp) < 1e-2
    assert abs(lk - lp) <= 1e-2 * abs(lp)
    assert rel(gk, gp) < 2e-2
    assert float(G["emb.word"].abs().sum()) > 0
    assert torch.count_nonzero(G["emb.word"][0]) == 0                 # the pad token never occurs
    assert torch.count_nonzero(G["emb.pos"][max(lens):]) == 0         # positions no token has
    assert torch.count_nonzero(G["emb.pos"][:max(lens)]) > 0


def _engine(packed, capture):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import tokens_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import BertBase
    cfg = FLConfig.for_world(1, model="bert", batch_size=8, samples_per_client=16, learning_rate=0.002,
                             cuda_graph=capture)
    shard = tokens_like(1, 16, seed=3, seq_len=256, min_len=64)[0]
    return GenericFedEngine(cfg, BertBase(shard.n_classes, layers=2, pad_id=0, packed=packed), shard,
                            rank=0, world=1, device=0)


def test_packed_bert_generic_engine_two_captured_rounds():
    eng = _engine(True, True)
    eng.capture()
    assert eng.graph_train is not None and not eng.capture_error
    for _ in range(2):
        eng.run_round()
    st = eng.read_state()
    assert math.isfinite(st["global_loss"])
    assert eng.drain_blocks() == [] and eng.host_ledger.verify_chain()


def test_packed_engine_round_matches_padded():
    """One eager round from the same seed: the global model moves by the same delta (rel < 5e-2;
    the two differ by bf16 rounding of GEMMs over a different row count)."""
    deltas = {}
    for packed in (False, True):
        eng = _engine(packed, False)
        before = eng.global_master.clone()
        eng.run_round()
        torch.cuda.synchronize()
        deltas[packed] = eng.global_master - before
        assert eng.drain_blocks() == []
        del eng
        torch.cuda.empty_cache()
    assert float(deltas[False].abs().sum()) > 0
    assert rel(deltas[True], deltas[False]) < 5e-2
