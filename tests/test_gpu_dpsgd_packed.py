"""DP-SGD on packed variable-length BERT on the H100: every segmented per-example kernel against fp64, against the
uniform kernel on each example alone (bit for bit) and with canaries, strided views and reruns; whole-vector
per-example norms of packed 2-layer BERT (full model and LoRA); the step's clipping, dropping and noise; packed
against padded DP-SGD; and captured packed LoRA engine rounds."""
import math

import numpy as np
import pytest
import torch

from bflc_demo_b200._native import C
from bflc_demo_b200.ops import dpsgd as D
from bflc_demo_b200.ops import nn as F
from bflc_demo_b200.protocol.oracle import DPSGD_SITE, dp_gauss

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
DEV = "cuda"
EDGES = [1, 63, 64, 65, 127, 128, 511, 512]


def _cu(lens):
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), device=DEV, dtype=torch.int32)
    seq = torch.repeat_interleave(torch.arange(len(lens), device=DEV, dtype=torch.int32),
                                  torch.tensor(lens, device=DEV))
    return cu, seq.to(torch.int32), [int(v) for v in cu.tolist()]


def _canaried(n):
    buf = torch.full((n + 2,), float("nan"), device=DEV)
    return buf, buf[1:-1]


def _ints(rows, cols, seed, lo=-1, hi=2, pad=0):
    """Small integers in a wider buffer: a strided, unaligned view when pad > 0."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = torch.randint(lo, hi, (rows, cols + pad), device=DEV, generator=g).to(BF)
    return w[:, pad // 2:pad // 2 + cols] if pad else w


def _canaries_intact(buf):
    assert torch.isnan(buf[0]) and torch.isnan(buf[-1])


# ------------------------------------------------------------------ kernels
def _gram(Q, R, bias, cu=None, **p):
    B = (cu.numel() - 1) if cu is not None else Q.shape[0] // R
    pairs = C().dpsgd_gram_pairs(R, True)
    buf, out = _canaried(pairs * B)
    C().dpsgd_pe_gram(Q, Q, R, bias, out, **({} if cu is None else {"cu_seqlens": cu}), **p)
    torch.cuda.synchronize()
    _canaries_intact(buf)
    return out.view(pairs, B).clone()


def _clip_sum(col):
    """k_dpsgd_clip's fp32 sum of an example's partials, in row order."""
    s = torch.zeros((), device=DEV)
    for v in col:
        s = s + v
    return s


@pytest.mark.parametrize("mode", ["dense", "onehot"])
def test_packed_gram_fp64_alone_canaries_strides_reruns(mode):
    cu, seq, h = _cu(EDGES)
    T = h[-1]
    Q = _ints(T, 136, 1, pad=10)                   # strided, unaligned
    if mode == "dense":
        p = dict(p1=_ints(T, 200, 2, pad=6), p2=None, mode=0)
        p["p2"] = p["p1"]
    else:
        ids = torch.randint(0, 40, (T,), device=DEV, dtype=torch.int32)
        p = dict(id1=ids, id2=ids, mode=1)
    bias = 1.0 if mode == "dense" else 0.0
    got = _gram(Q, 512, bias, cu, **p)
    assert torch.equal(got, _gram(Q, 512, bias, cu, **p))                     # reruns
    for n, L in enumerate(EDGES):
        sl = slice(h[n], h[n + 1])
        gq = Q[sl].double() @ Q[sl].double().t() + bias
        gp = (p["p1"][sl].double() @ p["p1"][sl].double().t() if mode == "dense" else
              (ids[sl][:, None] == ids[sl][None, :]).double())
        assert float(got[:, n].double().sum()) == float((gp * gq).sum()), L     # small integers: exact
        alone = _gram(Q[sl], L, bias, **{k: (v[sl] if torch.is_tensor(v) else v) for k, v in p.items()})
        pairs = C().dpsgd_gram_pairs(L, True)
        assert int((got[:, n] != 0).sum()) <= pairs
        assert torch.equal(_clip_sum(got[:, n]), _clip_sum(alone[:, 0])), L      # the design rule


def test_packed_gram_random_operands_match_each_example_alone_bit_for_bit():
    cu, seq, h = _cu([200, 5, 512, 65])
    g = torch.Generator(device=DEV).manual_seed(4)
    P = torch.randn(h[-1], 768, device=DEV, generator=g).to(BF)
    Q = torch.randn(h[-1], 3072, device=DEV, generator=g).to(BF)
    got = _gram(Q, 512, 1.0, cu, p1=P, p2=P, mode=0)
    for n, L in enumerate([200, 5, 512, 65]):
        sl = slice(h[n], h[n + 1])
        alone = _gram(Q[sl], L, 1.0, p1=P[sl], p2=P[sl], mode=0)
        nz = got[:, n][got[:, n] != 0]
        assert torch.equal(nz, alone[:, 0][alone[:, 0] != 0]), L      # the same partials, in the same order


def test_packed_norm_tiles_and_rows():
    cu, seq, h = _cu(EDGES)
    T = h[-1]
    A = _ints(T, 768, 5, pad=4)
    Bm = _ints(T, 8, 6, pad=8)
    tiles = C().dpsgd_norm_tiles(768, 8, False)
    buf, out = _canaried(tiles * len(EDGES))
    C().dpsgd_pe_norm(A, Bm, 512, out, cu_seqlens=cu)
    abuf, ab = _canaried(len(EDGES))
    C().dpsgd_pe_rows(A, Bm, 512, 1.0, None, ab, cu_seqlens=cu)
    torch.cuda.synchronize()
    _canaries_intact(buf)
    _canaries_intact(abuf)
    o1, a1 = out.clone(), ab.clone()
    C().dpsgd_pe_norm(A, Bm, 512, out, cu_seqlens=cu)
    C().dpsgd_pe_rows(A, Bm, 512, 1.0, None, ab, cu_seqlens=cu)
    assert torch.equal(o1, out) and torch.equal(a1, ab)
    sq = out.view(tiles, -1)
    for n, L in enumerate(EDGES):
        sl = slice(h[n], h[n + 1])
        assert float(sq[:, n].double().sum()) == float((A[sl].double().t() @ Bm[sl].double()).pow(2).sum())
        ref = float((A[sl].double().norm(dim=1) * (Bm[sl].double().pow(2).sum(1) + 1).sqrt()).sum())
        assert abs(float(ab[n]) - ref) <= 1e-5 * ref + 1e-6
        one, aone = torch.empty(tiles, device=DEV), torch.empty(1, device=DEV)
        C().dpsgd_pe_norm(A[sl], Bm[sl], L, one)
        C().dpsgd_pe_rows(A[sl], Bm[sl], L, 1.0, None, aone)
        assert torch.equal(one, sq[:, n]) and torch.equal(aone, ab[n:n + 1]), L


def _ln_inputs(rows, Cc, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(rows, Cc, device=DEV, generator=g).to(BF)
    dy = torch.randint(-3, 4, (rows, Cc), device=DEV, generator=g).to(BF)
    mean = x.float().mean(1).contiguous()
    rstd = (x.float().var(1, unbiased=False) + 1e-12).rsqrt().contiguous()
    return dy, x, mean, rstd


def test_packed_layer_norm_norms_and_release():
    cu, seq, h = _cu(EDGES)
    T, Cc, B = h[-1], 256, len(EDGES)
    dy, x, mean, rstd = _ln_inputs(T, Cc, 7)
    sbuf, sq = _canaried(B)
    abuf, ab = _canaried(B)
    C().dpsgd_pe_ln(dy, x, mean, rstd, 512, sq, ab, cu_seqlens=cu)
    torch.cuda.synchronize()
    _canaries_intact(sbuf)
    _canaries_intact(abuf)
    xh = (x.double() - mean.double()[:, None]) * rstd.double()[:, None]
    for n, L in enumerate(EDGES):
        sl = slice(h[n], h[n + 1])
        gg, gb = (dy[sl].double() * xh[sl]).sum(0), dy[sl].double().sum(0)
        want = float(gg.pow(2).sum() + gb.pow(2).sum())
        a = float((dy[sl].double().norm(dim=1) * (xh[sl].abs().max(1).values + 1)).sum())
        assert abs(float(sq[n]) - want) <= 1e-4 * a * a + 1e-4 * want
        s1, a1 = torch.empty(1, device=DEV), torch.empty(1, device=DEV)
        C().dpsgd_pe_ln(dy[sl], x[sl], mean[sl], rstd[sl], L, s1, a1)
        assert torch.equal(s1, sq[n:n + 1]) and torch.equal(a1, ab[n:n + 1]), L
    # the row scaling and the release: c[seq_ids[r]], a dropped example's rows skipped and written as +0
    c = torch.tensor([1.0, 0.5, 0.0, 1.0, 0.25, 1.0, 0.0, 0.5], device=DEV)
    Sbuf = torch.full((T + 2, Cc), float("nan"), device=DEV, dtype=BF)
    S = Sbuf[1:-1]
    C().dpsgd_scale_rows(dy, c, 1, S, seq_ids=seq)
    want = (dy.float() * c[seq.long()][:, None]).to(BF)
    assert torch.equal(S, want) and torch.isnan(Sbuf[0]).all() and torch.isnan(Sbuf[-1]).all()
    poisoned = x.clone()
    poisoned[h[2]:h[3]] = float("nan")                         # the dropped example's x need not be finite
    gg, gb = torch.zeros(Cc, device=DEV), torch.zeros(Cc, device=DEV)
    C().dpsgd_ln_release(S, poisoned, mean, rstd, c, 1, gg, gb, seq_ids=seq)
    keep = c[seq.long()] != 0
    assert torch.equal(gb.double(), S.double()[keep].sum(0))             # exact: small dyadic values
    xh32 = ((x.float() - mean[:, None]) * rstd[:, None]).double()
    assert torch.allclose(gg.double(), (S.double() * xh32)[keep].sum(0), rtol=1e-5, atol=1e-3)
    gg2, gb2 = torch.zeros(Cc, device=DEV), torch.zeros(Cc, device=DEV)
    C().dpsgd_ln_release(S, poisoned, mean, rstd, c, 1, gg2, gb2, seq_ids=seq)
    assert torch.equal(gg, gg2) and torch.equal(gb, gb2)


def test_bad_segmentation_drops_the_example():
    """cu values the host did not check (a length past max_len, cu[0] != 0) give a NaN partial, never a read
    past the example's rows: k_dpsgd_clip then drops the example."""
    cu, seq, h = _cu([100, 28])
    A, Bm = _ints(128, 256, 1), _ints(128, 256, 2)
    out = torch.zeros(C().dpsgd_gram_pairs(32, True) * 2, device=DEV)
    C().dpsgd_pe_gram(Bm, Bm, 32, 0.0, out, p1=A, p2=A, mode=0, cu_seqlens=cu)     # max_len 32: one tile
    assert torch.isnan(out[0]) and torch.isfinite(out[1])
    bad = cu + 1
    ab = torch.zeros(2, device=DEV)
    C().dpsgd_pe_rows(A, Bm, 64, 0.0, None, ab, cu_seqlens=bad)
    assert torch.isnan(ab).all()


# ------------------------------------------------------------------ whole models
LENS = [128, 100, 37, 5]


def _net(kind, dropout=0.0, packed=True):
    from bflc_demo_b200.models.lora import LoRANet
    from bflc_demo_b200.models.nets import BertBase
    base = BertBase(2, layers=2, pad_id=0, packed=packed, dropout=dropout)
    return LoRANet(base, 8, targets="q,v") if kind == "lora" else base


def _inputs(net, lens=LENS, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(len(lens), 256, dtype=torch.int64)
    for i, n in enumerate(lens):
        ids[i, :n] = torch.randint(1, 1000, (n,), generator=g)
    return net.preprocess(ids.to(DEV)), torch.randint(0, 2, (len(lens),), generator=g).to(DEV, torch.int32)


def _state(net, seed=3):
    P = net.spec.total
    master = torch.zeros(P, device=DEV)
    net.init_(master, seed=seed)
    return master, master.to(BF), torch.zeros(P, device=DEV)


def _seg(x):
    from bflc_demo_b200.data.packing import PackedTokens
    return x if isinstance(x, PackedTokens) else None


def _grad(net, x, y, state, dp=None, rng=None):
    master, shadow, grad = state
    grad.zero_()
    b = net.bind(master, shadow, grad)
    loss = net.loss(b, x, y, rng=rng) if rng is not None else net.loss(b, x, y)
    if dp is None:
        loss.backward()
    else:
        dp.begin(_seg(x))
        loss.backward()
        dp.finish(grad, 0)
    torch.cuda.synchronize()
    return grad.clone()


def _word():
    return torch.zeros(1, device=DEV, dtype=torch.int32)


def _snapshot(monkeypatch):
    fin = D.DPSGDStep.finish

    def spy(self, grad, add, n_valid=None):
        self._snap = list(self._records)
        return fin(self, grad, add, n_valid)

    monkeypatch.setattr(D.DPSGDStep, "finish", spy)


def _rows(lay, n):
    """Example n's rows of a record: an int R (uniform), or the packed step's segments (host offsets)."""
    if isinstance(lay, int):
        return slice(n * lay, (n + 1) * lay)
    return slice(lay.offsets[n] - lay.offsets[0], lay.offsets[n + 1] - lay.offsets[0])


def _per_example_fp64(dp, net, state, B):
    grad = state[2]
    out = torch.zeros(B, net.spec.total, dtype=torch.float64, device=DEV)
    base = grad.data_ptr()

    def put(n, g, val):
        off = (g.data_ptr() - base) // 4
        out[n, off:off + g.numel()].view(g.shape).add_(val)

    for rec in dp._snap:
        kind = rec[0]
        for n in range(B):
            if kind == "lin":
                _, dz, op, gw, gb, lay, _ = rec
                sl = _rows(lay, n)
                if gw is not None:
                    put(n, gw, dz[sl].double().t() @ op[sl].double())
                if gb is not None:
                    put(n, gb, dz[sl].double().sum(0))
            elif kind == "ln":
                _, dy, x, mean, rstd, gg, gb, lay = rec
                sl = _rows(lay, n)
                xh = ((x[sl].float() - mean[sl, None]) * rstd[sl, None]).double()
                if gg is not None:
                    put(n, gg, (dy[sl].double() * xh).sum(0))
                if gb is not None:
                    put(n, gb, dy[sl].double().sum(0))
            else:
                _, dy, ents, lay = rec
                sl = _rows(lay, n)
                for ids, g, _ in ents:
                    put(n, g, torch.zeros(g.shape, dtype=torch.float64, device=DEV).index_add_(
                        0, ids[sl].long(), dy[sl].double()))
    return out * B


@pytest.mark.parametrize("kind, dropout", [("full", 0.0), ("full", 0.1), ("lora", 0.0), ("lora", 0.1)])
def test_per_example_norms_match_fp64_over_the_whole_vector(kind, dropout, monkeypatch):
    from bflc_demo_b200.ops.nn import DropoutRNG
    _snapshot(monkeypatch)
    net = _net(kind, dropout)
    B = len(LENS)
    x, y = _inputs(net)
    state = _state(net)
    rng = DropoutRNG(11, _word()) if dropout > 0 else None
    dp = D.DPSGDStep(net.spec, B, 1e30, 0.0, 0, _word(), DEV)
    _grad(net, x, y, state, dp, rng)
    assert any(not isinstance(r[-1] if r[0] != "lin" else r[5], int) for r in dp._snap)   # segmented sites
    want = _per_example_fp64(dp, net, state, B).pow(2).sum(1) / B ** 2
    s = dp.sq[:dp._n_sq].double().sum(0)
    slack = (dp.kap[:dp._n_ab].double()[:, None] * dp.ab[:dp._n_ab].double() ** 2).sum(0)
    err = (s - want).abs()
    print(kind, dropout, "rel err", (err / want).tolist())
    assert (want > 0).all() and (err <= slack + 1e-3 * want).all(), (s, want, slack)


def test_unclipped_noiseless_packed_step_is_the_plain_packed_step(monkeypatch):
    _snapshot(monkeypatch)
    net = _net("full")
    B = len(LENS)
    x, y = _inputs(net)
    state = _state(net)
    dp = D.DPSGDStep(net.spec, B, 1e30, 0.0, 0, _word(), DEV)
    got = _grad(net, x, y, state, dp)
    assert torch.equal(got, _grad(net, x, y, state, dp))                      # bit-reproducible
    assert torch.equal(dp.c, torch.ones(B, device=DEV)) and int(dp.dropped) == 0
    col_abs = {r[4].data_ptr(): r[1].double().abs().sum(0) for r in dp._snap if r[0] == "lin" and r[4] is not None}
    monkeypatch.setattr(F, "_split_k", lambda *a: 1)
    plain = _grad(net, x, y, state)
    G_, P_, Gs = net.spec.views(got), net.spec.views(plain), net.spec.views(state[2])
    for e in net.spec.entries:
        a, b = G_[e.name].double(), P_[e.name].double()
        if len(e.shape) == 2 and not e.name.startswith("emb."):
            assert torch.equal(a, b), e.name
        else:
            ptr = Gs[e.name].data_ptr()
            tol = 2 ** -8 * col_abs[ptr] + 1e-7 if ptr in col_abs else 2 ** -12 * b.abs().max() + 1e-7
            assert ((a - b).abs() <= tol).all(), (e.name, float((a - b).abs().max()))


@pytest.mark.parametrize("kind", ["full", "lora"])
def test_clipped_packed_step_against_fp64_per_example_clipping(kind, monkeypatch):
    _snapshot(monkeypatch)
    net = _net(kind)
    B = len(LENS)
    x, y = _inputs(net, seed=4)
    state = _state(net)
    probe = D.DPSGDStep(net.spec, B, 1e30, 0.0, 0, _word(), DEV)
    _grad(net, x, y, state, probe)
    g = _per_example_fp64(probe, net, state, B)
    norms = g.norm(dim=1)
    clip = float(norms.median())
    dp = D.DPSGDStep(net.spec, B, clip, 0.0, 0, _word(), DEV)
    got = _grad(net, x, y, state, dp).double()
    c = dp.c.double()
    ideal = (clip / norms).clamp(max=1)
    assert (c < 1).any() and (c <= ideal * (1 + 1e-6)).all() and float((c / ideal).min()) > 0.5
    ref = (g * c[:, None]).sum(0) / B
    rel = float((got - ref).norm() / ref.norm())
    print(kind, "relative error of the clipped packed step", rel)
    assert rel < 2 ** -6


def test_single_example_contribution_is_within_the_clip():
    net = _net("full")
    x, y = _inputs(net, lens=[77], seed=6)
    state = _state(net)
    unclipped = _grad(net, x, y, state, D.DPSGDStep(net.spec, 1, 1e30, 0.0, 0, _word(), DEV))
    clip = 0.25 * float(unclipped.double().norm())
    n = float(_grad(net, x, y, state, D.DPSGDStep(net.spec, 1, clip, 0.0, 0, _word(), DEV)).double().norm())
    assert 0.3 * clip < n <= clip, (n, clip)


def test_non_finite_example_is_dropped_and_the_step_stays_finite(monkeypatch):
    rec = D.DPSGDStep.record_layernorm

    def poison(self, dy, x, mean, rstd, gg, gb):
        if self._seg is not None and dy.shape[0] == self._seg.T:
            dy[self._seg.offsets[2] + 5, 7] = float("nan")          # example 2's sixth token
        return rec(self, dy, x, mean, rstd, gg, gb)

    monkeypatch.setattr(D.DPSGDStep, "record_layernorm", poison)
    net = _net("full")
    x, y = _inputs(net, seed=8)
    state = _state(net)
    dp = D.DPSGDStep(net.spec, len(LENS), 1e30, 0.0, 0, _word(), DEV)
    got = _grad(net, x, y, state, dp)
    assert int(dp.dropped) == 1 and float(dp.c[2]) == 0.0 and torch.isfinite(got).all()
    assert float(got.abs().sum()) > 0


def test_noise_is_z_c_over_b():
    net = _net("lora")
    B = len(LENS)
    x, y = _inputs(net, seed=9)
    state = _state(net)
    clip, z, seed, add = 0.5, 2.0, 0xBEEF, 2
    word = torch.tensor([17], device=DEV, dtype=torch.int32)

    def step(noise):
        master, shadow, grad = state
        grad.zero_()
        loss = net.loss(net.bind(master, shadow, grad), x, y)
        dp = D.DPSGDStep(net.spec, B, clip, noise, seed, word, DEV)
        dp.begin(x)
        loss.backward()
        dp.finish(grad, add)
        torch.cuda.synchronize()
        return grad.clone()

    diff = (step(z).double() - step(0.0).double()).cpu()
    want = z * clip / B * torch.from_numpy(dp_gauss(seed, 17 + add, 0, net.spec.total, DPSGD_SITE)).double()
    assert float((diff - want).abs().max()) < 1e-6 * float(want.abs().max())


@pytest.mark.parametrize("kind", ["full", "lora"])
def test_packed_against_padded_dpsgd(kind, monkeypatch):
    """The same examples, seed and clip: packed and padded DP-SGD agree on the clip factors and the release to the
    tolerance of packed against padded BERT (bf16 GEMMs over different row counts)."""
    _snapshot(monkeypatch)
    out = {}
    for packed in (False, True):
        net = _net(kind, packed=packed)
        x, y = _inputs(net, seed=12)
        state = _state(net)
        probe = D.DPSGDStep(net.spec, len(LENS), 1e30, 0.0, 0, _word(), DEV)
        _grad(net, x, y, state, probe)
        out[packed] = (net, x, y, state, _per_example_fp64(probe, net, state, len(LENS)).norm(dim=1))
    clip = float(out[False][4].median())
    res = {}
    for packed, (net, x, y, state, _) in out.items():
        dp = D.DPSGDStep(net.spec, len(LENS), clip, 0.0, 0, _word(), DEV)
        res[packed] = (_grad(net, x, y, state, dp).double(), dp.c.double().clone())
    (gp, cp), (gk, ck) = res[False], res[True]
    assert (cp < 1).any()
    assert float(((ck - cp).abs() / cp).max()) < 2e-2, (ck, cp)
    assert float((gk - gp).norm() / gp.norm()) < 2e-2


# ------------------------------------------------------------------ engine rounds
def _engine(packed, capture, dpsgd=True):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import tokens_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.lora import LoRANet
    from bflc_demo_b200.models.nets import BertBase
    dp = dict(dpsgd_clip=0.5, dpsgd_noise=1.0, dpsgd_seed=3, dpsgd_packed=packed) if dpsgd else {}
    cfg = FLConfig.for_world(1, model="bert", batch_size=8, samples_per_client=16, learning_rate=0.002,
                             cuda_graph=capture, lora_rank=8, **dp)
    shard = tokens_like(1, 16, seed=3, seq_len=256, min_len=32)[0]
    base = BertBase(shard.n_classes, layers=2, pad_id=0, packed=packed)
    return GenericFedEngine(cfg, LoRANet(base, cfg.lora_rank, cfg.lora_alpha, cfg.lora_targets), shard,
                            rank=0, world=1, device=0)


def test_captured_packed_lora_dpsgd_rounds():
    eng = _engine(True, True)
    eng.capture()
    assert eng.graph_train is not None and not eng.capture_error
    for _ in range(3):
        eng.run_round()
    torch.cuda.synchronize()
    assert math.isfinite(eng.read_state()["global_loss"])
    assert eng.drain_blocks() == [] and eng.host_ledger.verify_chain()
    # capture() runs one round eagerly before it captures: three replays follow four eager rounds
    eager = _engine(True, False)
    for _ in range(4):
        eager.run_round()
    torch.cuda.synchronize()
    assert torch.equal(eng.global_master, eager.global_master)            # graph replay = eager, bit for bit
    padded = _engine(False, False)
    for _ in range(4):
        padded.run_round()
    torch.cuda.synchronize()
    eps, _ = eager.privacy_spent_local()
    assert math.isfinite(eps) and eps > 0
    assert padded.privacy_spent_local() == eager.privacy_spent_local() == eng.privacy_spent_local()


def test_packed_engine_round_matches_padded():
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
    assert float((deltas[True] - deltas[False]).norm() / deltas[False].norm()) < 5e-2


def test_engine_refuses_packed_dpsgd_without_the_opt_in():
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import tokens_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.lora import LoRANet
    from bflc_demo_b200.models.nets import BertBase
    cfg = FLConfig.for_world(1, model="bert", batch_size=8, samples_per_client=16, lora_rank=8, dpsgd_clip=0.5)
    shard = tokens_like(1, 16, seed=3, seq_len=128, min_len=32)[0]
    net = LoRANet(BertBase(2, layers=1, pad_id=0, packed=True), 8)
    with pytest.raises(ValueError, match="packed batches are not supported"):
        GenericFedEngine(cfg, net, shard, rank=0, world=1, device=0)
