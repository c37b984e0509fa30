"""Dropout in BERT training (csrc/include/philox.hpp): the exported attention keep masks against the
numpy Philox reference, the tiled / packed attention kernels with dropout against exact placements
and fp32 autograd, routing and bit-identity, repeatability under CUDA-graph replay and step-word
changes, the hidden dropout kernel, BertBase(dropout=...) and the generic engine."""
import math

import numpy as np
import pytest
import torch

from test_dropout_host import attention_keep_ref, hidden_keep_ref

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
D = 64
SEED = 0x1234_5678_9ABC_DEF0


def rel(x, ref):
    return ((x.float() - ref.float()).norm() / (ref.float().norm() + 1e-12)).item()


@pytest.fixture(scope="module")
def F():
    from bflc_demo_b200.ops import nn
    return nn


def _rng(F, step=5, add=0, seed=SEED):
    return F.DropoutRNG(seed, torch.tensor([step], device="cuda", dtype=torch.int32), add)


def _mask(B, H, S, p, rng, site):
    from bflc_demo_b200._native import C
    m = torch.empty(B * H, S, S, device="cuda", dtype=torch.uint8)
    C().dropout_keep_mask(m, B, H, S, p, rng.seed, rng.step, rng.add, site)
    return m.bool()


def _cu(lens):
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    return cu


# ------------------------------------------------------------------------------ exported masks
@pytest.mark.parametrize("B,H,S", [(2, 3, 64), (1, 2, 512), (3, 1, 200)])
def test_exported_mask_matches_numpy(F, B, H, S):
    rng = _rng(F, step=11, add=4)
    got = _mask(B, H, S, 0.1, rng, 7).cpu().numpy()
    assert np.array_equal(got, attention_keep_ref(SEED, 15, 7, 0.1, B, H, S))


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_keep_fraction(F, p):
    B, H, S = 4, 12, 512                           # 12.6 M elements
    m = _mask(B, H, S, p, _rng(F), 3)
    n = m.numel()
    frac = m.float().mean().item()
    sigma = math.sqrt(p * (1 - p) / n)
    assert abs(frac - (1 - p)) < 6 * sigma, (frac, 1 - p, sigma)


def test_masks_differ_across_sites_steps_heads_sequences(F):
    B, H, S = 2, 2, 128
    a = _mask(B, H, S, 0.5, _rng(F, step=1), 1)
    for other in (_mask(B, H, S, 0.5, _rng(F, step=1), 2), _mask(B, H, S, 0.5, _rng(F, step=2), 1),
                  _mask(B, H, S, 0.5, _rng(F, step=1, add=1), 1), _mask(B, H, S, 0.5, _rng(F, step=1, seed=9), 1)):
        assert (a != other).float().mean() > 0.4
    assert (a[0] != a[1]).float().mean() > 0.4     # heads of one sequence
    assert (a[0] != a[H]).float().mean() > 0.4     # sequences


# ------------------------------------------------------------------------------ exact placement
def _placement_inputs(B, S, H, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.zeros(B * S, H * D, device="cuda", dtype=BF).requires_grad_(True)
    k = torch.zeros(B * S, H * D, device="cuda", dtype=BF).requires_grad_(True)
    sign = lambda: (torch.randint(0, 2, (B * S, H * D), device="cuda", generator=g) * 2 - 1).to(BF)  # noqa: E731
    return q, k, sign().requires_grad_(True), sign()


@pytest.mark.parametrize("packed", [False, True])
def test_exact_placement(F, packed):
    """Q = K = 0: P = 1 / len on the keys of the sequence, so o_i = 1/(1-p) * sum of the kept V_j / len
    and dV_j = 1/(1-p) * sum of dO_i over the rows that keep j, / len.  The tolerance is below half of
    one element's contribution: a single misplaced keep decision fails."""
    p, H, S = 0.3, 2, 64
    lens = [64, 1, 37, 8, 50]
    B = len(lens)
    rng = _rng(F, step=3)
    z = 1.0 / (1.0 - p)
    q, k, v, do = _placement_inputs(B, S, H, 21)
    keep = attention_keep_ref(SEED, 3, 9, p, B, H, S)                # [B*H, S, S]
    real = torch.zeros(B * S, dtype=torch.bool, device="cuda")
    for b, n in enumerate(lens):
        real[b * S:b * S + n] = True
    if packed:
        do = do * real[:, None]                                      # padded rows carry no gradient
        qp, kp, vp = (t.detach()[real].clone().requires_grad_(True) for t in (q, k, v))
        cu = torch.tensor(_cu(lens), device="cuda", dtype=torch.int32)
        o = F.attention_packed(qp, kp, vp, cu, max(lens), H, dropout_p=p, rng=rng, site=9)
        o.backward(do[real])
        o_full = torch.zeros(B * S, H * D, device="cuda")
        dv_full = torch.zeros(B * S, H * D, device="cuda")
        o_full[real], dv_full[real] = o.detach().float(), vp.grad.float()
    else:
        lengths = torch.tensor(lens, device="cuda", dtype=torch.int32)
        o = F.attention(q, k, v, B, S, H, lengths=lengths, dropout_p=p, rng=rng, site=9)
        o.backward(do)
        o_full, dv_full = o.detach().float(), v.grad.float()
    V, dO = v.detach().float(), do.float()
    for b, n in enumerate(lens):
        rows = slice(b * S, b * S + S)
        qrows = n if packed else S                                   # padded query rows are computed too
        for h in range(H):
            kh = torch.from_numpy(keep[b * H + h]).cuda().float()[:, :n]     # [i, j < n]
            cols = slice(h * D, h * D + D)
            o_ref = z * kh[:qrows] @ V[rows][:n, cols] / n
            dv_ref = z * kh[:qrows].t() @ dO[rows][:qrows, cols] / n
            tol = 0.5 * z / n
            assert (o_full[rows][:qrows, cols] - o_ref).abs().max() < tol, (b, h)
            assert (dv_full[rows][:n, cols] - dv_ref).abs().max() < tol, (b, h)


# ------------------------------------------------------------------------------ fp32 reference
def _ref(q, k, v, do, B, S, H, lens, keep, p):
    """fp32 autograd of ((softmax with key mask) * keep / (1 - p)) V, heads [B, H, S, D]."""
    def heads(t):
        return t.detach().float().view(B, S, H, D).permute(0, 2, 1, 3).requires_grad_(True)
    qh, kh, vh = heads(q), heads(k), heads(v)
    s = qh @ kh.transpose(-1, -2) / math.sqrt(D)
    km = torch.arange(S, device="cuda")[None, :] < torch.tensor(lens, device="cuda")[:, None]
    s = s.masked_fill(~km[:, None, None, :], float("-inf"))
    P = torch.softmax(s, -1)
    Z = torch.from_numpy(keep).cuda().view(B, H, S, S).float() / (1 - p)
    o = (P * Z) @ vh
    o.backward(do.float().view(B, S, H, D).permute(0, 2, 1, 3))
    back = lambda t: t.permute(0, 2, 1, 3).reshape(B * S, H * D)  # noqa: E731
    return back(o.detach()), back(qh.grad), back(kh.grad), back(vh.grad)


@pytest.mark.parametrize("S,lens", [(64, [64, 30]), (128, [128, 128]), (128, [100, 7]), (256, [256, 131]),
                                    (512, [512, 300])])
def test_padded_matches_fp32_reference(F, S, lens):
    H, p, B = 2, 0.1, len(lens)
    g = torch.Generator(device="cuda").manual_seed(S)
    q, k, v = [(torch.randn(B * S, H * D, device="cuda", generator=g) * 0.7).to(BF).requires_grad_(True)
               for _ in range(3)]
    do = torch.randn(B * S, H * D, device="cuda", generator=g).to(BF)
    rng = _rng(F, step=17)
    lengths = None if all(n == S for n in lens) else torch.tensor(lens, device="cuda", dtype=torch.int32)
    o = F.attention(q, k, v, B, S, H, lengths=lengths, dropout_p=p, rng=rng, site=4)
    o.backward(do)
    keep = _mask(B, H, S, p, rng, 4).cpu().numpy()
    ro, rq, rk, rv = _ref(q, k, v, do, B, S, H, lens, keep, p)
    assert rel(o, ro) < 2e-2
    assert rel(q.grad, rq) < 5e-2 and rel(k.grad, rk) < 5e-2 and rel(v.grad, rv) < 5e-2


def test_packed_matches_fp32_reference(F):
    H, p = 2, 0.1
    lens = [1, 63, 64, 65, 129, 300, 512]
    B, S, cu = len(lens), 512, _cu(lens)
    g = torch.Generator(device="cuda").manual_seed(5)
    padded = [(torch.randn(B * S, H * D, device="cuda", generator=g) * 0.7).to(BF) for _ in range(3)]
    do = torch.randn(B * S, H * D, device="cuda", generator=g).to(BF)
    real = torch.zeros(B * S, dtype=torch.bool, device="cuda")
    for b, n in enumerate(lens):
        real[b * S:b * S + n] = True
    do[~real] = 0
    qp, kp, vp = (t[real].clone().requires_grad_(True) for t in padded)
    rng = _rng(F, step=2)
    o = F.attention_packed(qp, kp, vp, torch.tensor(cu, device="cuda", dtype=torch.int32), max(lens), H,
                           dropout_p=p, rng=rng, site=6)
    o.backward(do[real])
    keep = _mask(B, H, S, p, rng, 6).cpu().numpy()
    refs = _ref(*padded, do, B, S, H, lens, keep, p)
    assert rel(o, refs[0][real]) < 2e-2
    for got, r in zip((qp.grad, kp.grad, vp.grad), refs[1:]):
        assert rel(got, r[real]) < 5e-2


# ------------------------------------------------------------------------------ routing, bit identity
def _run(F, q, k, v, do, **kw):
    for t in (q, k, v):
        t.grad = None
    o = F.attention(q, k, v, **kw)
    o.backward(do)
    return [o.detach().clone(), q.grad.clone(), k.grad.clone(), v.grad.clone()]


@pytest.mark.parametrize("S,masked", [(128, False), (128, True), (256, True)])
def test_p_zero_is_bit_identical(F, S, masked):
    B, H = 3, 2
    q, k, v = [(torch.randn(B * S, H * D, device="cuda") * 0.7).to(BF).requires_grad_(True) for _ in range(3)]
    do = torch.randn(B * S, H * D, device="cuda").to(BF)
    lengths = torch.tensor([S, 70, 3], device="cuda", dtype=torch.int32) if masked else None
    a = _run(F, q, k, v, do, B=B, S=S, H=H, lengths=lengths)
    b = _run(F, q, k, v, do, B=B, S=S, H=H, lengths=lengths, dropout_p=0.0, rng=_rng(F), site=3)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_packed_and_padded_bit_identical_with_dropout(F):
    S, H, p = 256, 2, 0.1
    lens = [1, 63, 64, 65, 129, 256, 200]
    B, cu = len(lens), _cu(lens)
    g = torch.Generator(device="cuda").manual_seed(9)
    padded = [(torch.randn(B * S, H * D, device="cuda", generator=g) * 0.7).to(BF) for _ in range(3)]
    do_p = torch.randn(B * S, H * D, device="cuda", generator=g).to(BF)
    real = torch.zeros(B * S, dtype=torch.bool, device="cuda")
    for b, n in enumerate(lens):
        real[b * S:b * S + n] = True
    do_p[~real] = 0
    packed = [t[real].clone().requires_grad_(True) for t in padded]
    padded = [t.requires_grad_(True) for t in padded]
    rng = _rng(F, step=8)
    ref = _run(F, *padded, do_p, B=B, S=S, H=H, lengths=torch.tensor(lens, device="cuda", dtype=torch.int32),
               dropout_p=p, rng=rng, site=5)
    for t in packed:
        t.grad = None
    o = F.attention_packed(*packed, torch.tensor(cu, device="cuda", dtype=torch.int32), max(lens), H,
                           dropout_p=p, rng=rng, site=5)
    o.backward(do_p[real])
    for name, a, b in zip(("o", "dq", "dk", "dv"), [o.detach()] + [t.grad for t in packed], ref):
        assert torch.equal(a, b[real]), f"{name}: max |d| = {(a.float() - b[real].float()).abs().max().item()}"


def test_dropout_argument_checks(F):
    q, k, v = [torch.zeros(128, 2 * D, device="cuda", dtype=BF) for _ in range(3)]
    with pytest.raises(ValueError):
        F.attention(q, k, v, 1, 128, 2, dropout_p=0.1)                       # no rng
    with pytest.raises(ValueError):
        F.attention(q, k, v, 1, 128, 2, dropout_p=1.0, rng=_rng(F))
    with pytest.raises(ValueError):
        F.attention(q, k, v, 1, 128, 2, fused=False, dropout_p=0.1, rng=_rng(F))
    q3 = torch.zeros(96, 2 * D, device="cuda", dtype=BF)
    with pytest.raises(ValueError):
        F.attention(q3, q3, q3, 1, 96, 2, dropout_p=0.1, rng=_rng(F))        # unsupported shape
    with pytest.raises(ValueError):
        F.attention_packed(q, k, v, torch.tensor([0, 128], device="cuda", dtype=torch.int32), 128, 2,
                           dropout_p=-0.1, rng=_rng(F))


# ------------------------------------------------------------------------------ repeatability
def test_deterministic_graph_replay_and_step_word(F):
    B, S, H, p = 4, 256, 3, 0.1
    q, k, v = [(torch.randn(B * S, H * D, device="cuda") * 0.7).to(BF).requires_grad_(True) for _ in range(3)]
    do = torch.randn(B * S, H * D, device="cuda").to(BF)
    lengths = torch.tensor([256, 100, 1, 64], device="cuda", dtype=torch.int32)
    rng = _rng(F, step=40, add=2)
    kw = dict(B=B, S=S, H=H, lengths=lengths, dropout_p=p, rng=rng, site=2)
    first, second = _run(F, q, k, v, do, **kw), _run(F, q, k, v, do, **kw)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    g = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        _run(F, q, k, v, do, **kw)
        with torch.cuda.graph(g, stream=st):
            for t in (q, k, v):
                t.grad = None
            o = F.attention(q, k, v, **kw)
            o.backward(do)
    torch.cuda.current_stream().wait_stream(st)
    g.replay()
    torch.cuda.synchronize()
    replay = lambda: [o.clone(), q.grad.clone(), k.grad.clone(), v.grad.clone()]  # noqa: E731
    for a, b in zip(first, replay()):
        assert torch.equal(a, b)
    rng.step.fill_(41)                              # a new step word: new masks, new results
    g.replay()
    torch.cuda.synchronize()
    changed = replay()
    assert not torch.equal(changed[0], first[0]) and not torch.equal(changed[3], first[3])
    rng.step.fill_(40)                              # restored: the first results, bit for bit
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(first, replay()):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------ hidden dropout
@pytest.mark.parametrize("packed", [False, True])
def test_hidden_dropout_exact(F, packed):
    p, C, S = 0.1, 768, 64
    lens = [64, 5, 33]
    rng = _rng(F, step=6, add=1)
    if packed:
        seq = torch.cat([torch.full((n,), b, dtype=torch.int32) for b, n in enumerate(lens)]).cuda()
        pos = torch.cat([torch.arange(n, dtype=torch.int32) for n in lens]).cuda()
        rows, kw = len(seq), dict(seq_ids=seq, pos_ids=pos)
        seq_np, pos_np = seq.cpu().numpy(), pos.cpu().numpy()
    else:
        rows, kw = len(lens) * S, dict(S=S)
        seq_np, pos_np = np.arange(rows) // S, np.arange(rows) % S
    x = torch.zeros(rows, C, device="cuda", dtype=BF, requires_grad=True)
    z = torch.ones(rows, C, device="cuda", dtype=BF, requires_grad=True)
    y = F.dropout_add(x, z, p, rng, 12, **kw)
    keep = torch.from_numpy(hidden_keep_ref(SEED, 7, 12, p, seq_np, pos_np, C)).cuda()
    one = torch.ones((), device="cuda")
    zs = torch.where(keep, one / (one - torch.tensor(p, device="cuda")), 0.0)   # keep / (1 - p), fp32
    want = zs.to(BF)
    assert torch.equal(y.detach(), want)
    dy = torch.randn(rows, C, device="cuda").to(BF)
    y.backward(dy)
    assert torch.equal(x.grad, dy)
    assert torch.equal(z.grad, (dy.float() * zs).to(BF))
    y2 = F.dropout(z.detach(), p, rng, 12, **kw)
    assert torch.equal(y2, want)


def test_hidden_dropout_packed_equals_padded(F):
    """Rows of a packed batch draw what the same rows of the right-padded batch draw."""
    p, C, S = 0.5, 256, 128
    lens = [128, 3, 77]
    rng = _rng(F, step=1)
    z = torch.randn(len(lens) * S, C, device="cuda").to(BF)
    real = torch.zeros(len(lens) * S, dtype=torch.bool, device="cuda")
    for b, n in enumerate(lens):
        real[b * S:b * S + n] = True
    seq = torch.cat([torch.full((n,), b, dtype=torch.int32) for b, n in enumerate(lens)]).cuda()
    pos = torch.cat([torch.arange(n, dtype=torch.int32) for n in lens]).cuda()
    a = F.dropout(z, p, rng, 3, S=S)[real]
    b = F.dropout(z[real].contiguous(), p, rng, 3, seq_ids=seq, pos_ids=pos)
    assert torch.equal(a, b)


# ------------------------------------------------------------------------------ BertBase
def _bert(packed, dropout, layers=2, pad_id=0):
    from bflc_demo_b200.models.nets import BertBase
    net = BertBase(2, layers=layers, pad_id=pad_id, packed=packed, dropout=dropout)
    master = torch.empty(net.spec.total)
    net.init_(master, seed=1)
    master = master.cuda()
    grad = torch.zeros_like(master)
    return net, net.bind(master, master.to(BF), grad), grad


def _ids(lens, S):
    torch.manual_seed(11)
    ids = torch.zeros(len(lens), S, dtype=torch.int64, device="cuda")
    for i, n in enumerate(lens):
        ids[i, :n] = torch.randint(1, 30522, (n,), device="cuda")
    return ids


def test_bert_eval_unchanged_and_training_drops(F):
    lens, S = [128, 100, 37, 5], 128
    ids = _ids(lens, S)
    y = torch.tensor([0, 1, 1, 0], device="cuda", dtype=torch.int32)
    net0, b0, _ = _bert(False, 0.0)
    net1, b1, _ = _bert(False, 0.1)
    x = net0.preprocess(ids)
    with torch.no_grad():
        assert torch.equal(net0.features(b0, x, False), net1.features(b1, x, False))
        assert torch.equal(net0.features(b0, x, True), net1.features(b1, x, True))     # no rng: no dropout
    assert torch.equal(net0.correct(b0, x, y), net1.correct(b1, x, y))
    rng = _rng(F, step=0)
    losses = []
    for step in (0, 1, 0):
        rng.step.fill_(step)
        with torch.no_grad():
            losses.append(float(net1.loss(b1, x, y, rng=rng)))
    assert losses[0] != losses[1] and losses[0] == losses[2]
    with torch.no_grad():
        assert float(net0.loss(b0, x, y, rng=rng)) != losses[0]        # dropout changes the loss


def test_bert_dropout_packed_matches_padded(F):
    lens, S = [128, 100, 37, 5], 256
    ids = _ids(lens, S)
    y = torch.tensor([0, 1, 1, 0], device="cuda", dtype=torch.int32)
    out = {}
    for packed in (False, True):
        net, b, grad = _bert(packed, 0.1)
        x = net.preprocess(ids)
        loss = net.loss(b, x, y, rng=_rng(F, step=3))
        loss.backward()
        torch.cuda.synchronize()
        out[packed] = (float(loss.detach()), grad.clone(), net.spec.views(grad))
    (lp, gp, Gp), (lk, gk, G) = out[False], out[True]
    assert abs(lk - lp) <= 1e-2 * abs(lp)
    assert rel(gk, gp) < 2e-2
    for Gx in (Gp, G):
        assert torch.count_nonzero(Gx["emb.word"][0]) == 0              # the pad token
        assert torch.count_nonzero(Gx["emb.pos"][max(lens):]) == 0      # positions no token has


# ------------------------------------------------------------------------------ engine
def _engine(lr, capture=True):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import tokens_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import BertBase
    cfg = FLConfig.for_world(1, model="bert", batch_size=8, samples_per_client=16, learning_rate=lr or 1e-3,
                             cuda_graph=capture)
    shard = tokens_like(1, 16, seed=3, seq_len=128, min_len=64)[0]
    eng = GenericFedEngine(cfg, BertBase(shard.n_classes, layers=2, pad_id=0, dropout=0.1), shard,
                           rank=0, world=1, device=0)
    eng.cfg.learning_rate = lr                      # 0: frozen weights (the config itself insists on lr > 0)
    return eng


def test_engine_two_captured_rounds_with_dropout():
    eng = _engine(0.002)
    eng.capture()
    assert eng.graph_train is not None and not eng.capture_error
    for _ in range(2):
        eng.run_round()
    st = eng.read_state()
    assert math.isfinite(st["global_loss"])
    assert eng.drain_blocks() == [] and eng.host_ledger.verify_chain()


def test_engine_replays_draw_new_masks_from_the_step_word():
    """lr = 0: the weights never move, so the training graph's loss changes only with the masks."""
    eng = _engine(0.0)
    eng.capture()
    assert eng.graph_train is not None
    word = eng.opt_step_word.clone()

    def replay():
        with torch.cuda.stream(eng.stream):
            eng.loss_sum.zero_()
            eng.graph_train.replay()
        eng.stream.synchronize()
        return eng.loss_sum.clone()

    first = replay()
    eng.opt_step_word.add_(eng.steps)               # what fed_plan_round does between rounds
    second = replay()
    assert not torch.equal(first, second)
    eng.opt_step_word.copy_(word)
    assert torch.equal(replay(), first)
    assert math.isfinite(float(first))
