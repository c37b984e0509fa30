"""Full-model DP-SGD on the H100: the Gram-form norm kernel (dense, one-hot and gather modes) against fp64,
the layer-norm norm kernel, the fixed-order layer-norm and embedding releases, and full BERT / GPT steps
and engine rounds with every parameter clipped."""
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
GPT_SMALL = dict(layers=2, hidden=128, heads=2, ffn=256, vocab=512, max_pos=128)


def _canaried(n):
    buf = torch.full((n + 2,), float("nan"), device=DEV)
    return buf, buf[1:-1]


def _gram_ref(P1, P2, Q1, Q2, R, bias, mode="dense", ids1=None, ids2=None):
    """fp64 sum_{t,t'} Gp Gq per example (and sum_t ||p_t|| ||q_t|| for the tolerance)."""
    B = Q1.shape[0] // R
    out, ab = [], []
    for n in range(B):
        sl = slice(n * R, (n + 1) * R)
        gq = Q1[sl].double() @ Q2[sl].double().t() + bias
        if mode == "dense":
            gp = P1[sl].double() @ P2[sl].double().t()
        elif mode == "onehot":
            gp = (ids1[sl][:, None] == ids2[sl][None, :]).double()
        else:
            gp = P1[sl].double()[:, ids2[sl].long()]
        out.append(float((gp * gq).sum()))
        pn = P1[sl].double().norm(dim=1) if mode != "onehot" else torch.ones(R, device=DEV, dtype=torch.float64)
        qn = (Q1[sl].double().pow(2).sum(1) + bias).sqrt()
        ab.append(float((pn * qn).sum()))
    return np.array(out), np.array(ab)


def _run_gram(Q1, Q2, R, bias, sym=True, **p):
    B = Q1.shape[0] // R
    pairs = C().dpsgd_gram_pairs(R, sym)
    buf, out = _canaried(pairs * B)
    C().dpsgd_pe_gram(Q1, Q2, R, bias, out, sym=sym, **p)
    torch.cuda.synchronize()
    assert torch.isnan(buf[0]) and torch.isnan(buf[-1])
    return out.view(pairs, B).double().sum(0).cpu().numpy(), out.clone()


# ------------------------------------------------------------------ the Gram kernel
@pytest.mark.parametrize("R, wp, wq, bias, B", [
    (64, 200, 768, 0.0, 1), (128, 768, 768, 1.0, 3), (192, 3072, 768, 1.0, 3), (512, 768, 200, 0.0, 1),
    (128, 8192, 768, 0.0, 16), (128, 768, 3072, 1.0, 16), (100, 200, 200, 1.0, 3)])
def test_gram_dense_against_fp64_with_canaries_and_reruns(R, wp, wq, bias, B):
    g = torch.Generator(device=DEV).manual_seed(R + wp + B)
    P = torch.randn(B * R, wp, device=DEV, generator=g).to(BF)
    Q = torch.randn(B * R, wq, device=DEV, generator=g).to(BF)
    got, raw = _run_gram(Q, Q, R, bias, p1=P, p2=P, mode=0)
    want, ab = _gram_ref(P, P, Q, Q, R, bias)
    kap = float(D.gram_kappa(wp, wq + 1, 64 + C().dpsgd_gram_pairs(R, True)))
    assert (np.abs(got - want) <= kap * ab ** 2).all(), (got, want)
    assert torch.equal(raw, _run_gram(Q, Q, R, bias, p1=P, p2=P, mode=0)[1])


def test_gram_is_exact_on_integers_and_reads_strided_views():
    g = torch.Generator(device=DEV).manual_seed(1)
    R, B = 96, 3
    Pw = torch.randint(-2, 3, (B * R, 208), device=DEV, generator=g).to(BF)
    Qw = torch.randint(-2, 3, (B * R, 136), device=DEV, generator=g).to(BF)
    P, Q = Pw[:, 3:203], Qw[:, 5:133]           # unaligned, strided views
    got, _ = _run_gram(Q, Q, R, 1.0, p1=P, p2=P, mode=0)
    want, _ = _gram_ref(P, P, Q, Q, R, 1.0)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("kind", ["equal", "distinct", "padding"])
def test_gram_one_hot_mode(kind):
    R, B, H = 128, 3, 768
    g = torch.Generator(device=DEV).manual_seed(2)
    if kind == "equal":
        ids = torch.full((B * R,), 7, device=DEV, dtype=torch.int32)
    elif kind == "distinct":
        ids = torch.arange(B * R, device=DEV, dtype=torch.int32)
    else:
        ids = torch.zeros(B * R, device=DEV, dtype=torch.int32)
        ids.view(B, R)[:, :10] = torch.randint(1, 50, (B, 10), device=DEV, generator=g, dtype=torch.int32)
    dy = torch.randint(-3, 4, (B * R, H), device=DEV, generator=g).to(BF)
    got, _ = _run_gram(dy, dy, R, 0.0, id1=ids, id2=ids, mode=1)
    want, _ = _gram_ref(None, None, dy, dy, R, 0.0, "onehot", ids, ids)
    assert np.array_equal(got, want)               # small integers: every sum is exact in fp32
    # the definition: ||sum_t e_{id_t} dy_t^T||^2, repeated ids counting
    for n in range(B):
        G = torch.zeros(B * R, H, dtype=torch.float64, device=DEV)
        G.index_add_(0, ids[n * R:(n + 1) * R].long(), dy[n * R:(n + 1) * R].double())
        assert float(G.pow(2).sum()) == got[n]


def test_gram_gather_mode_is_the_tied_cross_term():
    R, B, V, H = 128, 2, 512, 128
    g = torch.Generator(device=DEV).manual_seed(3)
    dl = torch.randint(-2, 3, (B * R, V), device=DEV, generator=g).to(BF)
    h = torch.randint(-2, 3, (B * R, H), device=DEV, generator=g).to(BF)
    dy = torch.randint(-2, 3, (B * R, H), device=DEV, generator=g).to(BF)
    ids = torch.randint(0, V, (B * R,), device=DEV, generator=g, dtype=torch.int32)
    got, _ = _run_gram(h, dy, R, 0.0, sym=False, p1=dl, id2=ids, mode=2)
    want, _ = _gram_ref(dl, None, h, dy, R, 0.0, "gather", None, ids)
    assert np.array_equal(got, 2 * want)


# ------------------------------------------------------------------ layer norms
def _ln_inputs(rows, Cc, seed, integer=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(rows, Cc, device=DEV, generator=g).to(BF)
    dy = (torch.randint(-3, 4, (rows, Cc), device=DEV, generator=g) if integer else
          torch.randn(rows, Cc, device=DEV, generator=g)).to(BF)
    mean = x.float().mean(1)
    rstd = (x.float().var(1, unbiased=False) + 1e-12).rsqrt()
    return dy, x, mean.contiguous(), rstd.contiguous()


@pytest.mark.parametrize("R, B", [(1, 16), (128, 3), (512, 1)])
def test_pe_ln_against_fp64(R, B):
    Cc = 768
    dy, x, mean, rstd = _ln_inputs(B * R, Cc, R)
    sq = torch.full((B,), float("nan"), device=DEV)
    ab = torch.full((B,), float("nan"), device=DEV)
    C().dpsgd_pe_ln(dy, x, mean, rstd, R, sq, ab)
    xh = (x.double() - mean.double()[:, None]) * rstd.double()[:, None]
    for n in range(B):
        sl = slice(n * R, (n + 1) * R)
        gg, gb = (dy[sl].double() * xh[sl]).sum(0), dy[sl].double().sum(0)
        want = float(gg.pow(2).sum() + gb.pow(2).sum())
        a = float((dy[sl].double().norm(dim=1) * (xh[sl].abs().max(1).values + 1)).sum())
        assert abs(float(sq[n]) - want) <= 1e-4 * a * a + 1e-4 * want
        assert abs(float(ab[n]) - a) <= 1e-5 * a


def test_fixed_order_releases_are_exact_and_bit_reproducible():
    R, B, Cc, V = 64, 4, 256, 40
    dy, x, mean, rstd = _ln_inputs(B * R, Cc, 5, integer=True)
    c = torch.tensor([1.0, 0.0, 1.0, 1.0], device=DEV)
    S = torch.empty_like(dy)
    C().dpsgd_scale_rows(dy, c, R, S)

    def ln():
        gg, gb = torch.zeros(Cc, device=DEV), torch.zeros(Cc, device=DEV)
        C().dpsgd_ln_release(S, x, mean, rstd, c, R, gg, gb)
        return gg, gb

    gg, gb = ln()
    keep = c.repeat_interleave(R).bool()
    assert torch.equal(gb.double(), dy.double()[keep].sum(0))          # small integers: exact
    xh = ((x.float() - mean[:, None]) * rstd[:, None]).double()
    assert torch.allclose(gg.double(), (dy.double() * xh)[keep].sum(0), rtol=1e-5, atol=1e-4)
    assert all(torch.equal(a, b) for a, b in zip((gg, gb), ln()))

    ids = torch.randint(0, V, (B * R,), device=DEV, dtype=torch.int32)
    ids[:50] = 3                                                       # a long run of one id

    def emb():
        G = torch.zeros(V, Cc, device=DEV)
        C().dpsgd_emb_release(S, ids, torch.empty_like(ids), G)
        return G

    G = emb()
    want = torch.zeros(V, Cc, dtype=torch.float64, device=DEV).index_add_(0, ids.long(), S.double())
    assert torch.equal(G.double(), want) and torch.equal(G, emb())


# ------------------------------------------------------------------ full models
def _net(kind, dropout=0.0):
    from bflc_demo_b200.models.nets import GPT, BertBase
    if kind == "gpt":
        return GPT(**GPT_SMALL, dropout=dropout), 4
    return BertBase(2, layers=2, pad_id=0 if kind == "bert_pad" else None, dropout=dropout), 4


def _inputs(kind, net, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    if kind == "gpt":
        ids = torch.randint(0, 512, (B, 128), generator=g)
        return net.preprocess(ids.to(DEV)), torch.randint(0, 512, (B, 128), generator=g).to(DEV, torch.int32)
    ids = torch.randint(1, 1000, (B, 128), generator=g)
    if kind == "bert_pad":
        for n in range(B):
            ids[n, 32 + 16 * n:] = 0
    return net.preprocess(ids.to(DEV)), torch.randint(0, 2, (B,), generator=g).to(DEV, torch.int32)


def _state(net, seed=3):
    P = net.spec.total
    master = torch.zeros(P, device=DEV)
    net.init_(master, seed=seed)
    return master, master.to(BF), torch.zeros(P, device=DEV)


def _grad(net, x, y, state, dp=None, rng=None):
    master, shadow, grad = state
    grad.zero_()
    b = net.bind(master, shadow, grad)
    loss = net.loss(b, x, y, rng=rng) if rng is not None else net.loss(b, x, y)
    if dp is None:
        loss.backward()
    else:
        dp.begin()
        loss.backward()
        dp.finish(grad, 0)
    torch.cuda.synchronize()
    return grad.clone()


def _word():
    return torch.zeros(1, device=DEV, dtype=torch.int32)


def _per_example_fp64(dp, net, state, B):
    """Each example's gradient over the whole flat vector in fp64, materialised from the recorded sites
    (weight gradients dz_n^T (x_n, 1), layer-norm sums, embedding row sums; a tied table's two uses add
    into one parameter), times B (the recorded rows are of the batch-mean loss)."""
    grad = state[2]
    out = torch.zeros(B, net.spec.total, dtype=torch.float64, device=DEV)
    base = grad.data_ptr()

    def put(n, g, val):
        off = (g.data_ptr() - base) // 4
        if g.dim() == 2:
            out[n, off:off + g.numel()].view(g.shape).add_(val)
        else:
            out[n, off:off + g.numel()].add_(val)

    for rec in dp._snap:
        kind = rec[0]
        for n in range(B):
            if kind == "lin":
                _, dz, op, gw, gb, R, _ = rec
                sl = slice(n * R, (n + 1) * R)
                if gw is not None:
                    put(n, gw, dz[sl].double().t() @ op[sl].double())
                if gb is not None:
                    put(n, gb, dz[sl].double().sum(0))
            elif kind == "ln":
                _, dy, x, mean, rstd, gg, gb, R = rec
                sl = slice(n * R, (n + 1) * R)
                xh = ((x[sl].float() - mean[sl, None]) * rstd[sl, None]).double()
                if gg is not None:
                    put(n, gg, (dy[sl].double() * xh).sum(0))
                if gb is not None:
                    put(n, gb, dy[sl].double().sum(0))
            else:
                _, dy, ents, R = rec
                sl = slice(n * R, (n + 1) * R)
                for ids, g, _ in ents:
                    put(n, g, torch.zeros(g.shape, dtype=torch.float64, device=DEV).index_add_(
                        0, ids[sl].long(), dy[sl].double()))
    return out * B


def _snapshot(monkeypatch):
    fin = D.DPSGDStep.finish

    def spy(self, grad, add):
        self._snap = list(self._records)
        return fin(self, grad, add)

    monkeypatch.setattr(D.DPSGDStep, "finish", spy)


@pytest.mark.parametrize("kind, dropout", [("bert", 0.0), ("bert_pad", 0.0), ("bert_pad", 0.1), ("gpt", 0.0)])
def test_per_example_norms_match_fp64_over_the_whole_vector(kind, dropout, monkeypatch):
    """sum sq over every site (the Gram partials, one-hot embeddings, the tied cross term, layer norms,
    one-row sites) equals each example's fp64 squared norm within the certified slack sum kappa ab^2."""
    from bflc_demo_b200.ops.nn import DropoutRNG
    _snapshot(monkeypatch)
    net, B = _net(kind, dropout)
    x, y = _inputs(kind, net, B)
    state = _state(net)
    rng = DropoutRNG(11, _word()) if dropout > 0 else None
    dp = D.DPSGDStep(net.spec, B, 1e30, 0.0, 0, _word(), DEV)
    _grad(net, x, y, state, dp, rng)
    g = _per_example_fp64(dp, net, state, B)
    want = g.pow(2).sum(1) / B ** 2
    s = dp.sq[:dp._n_sq].double().sum(0)
    slack = (dp.kap[:dp._n_ab].double()[:, None] * dp.ab[:dp._n_ab].double() ** 2).sum(0)
    assert dp._kappa and (slack > 0).all()
    err = (s - want).abs()
    print(kind, dropout, "rel err", (err / want).tolist(), "slack / s", (slack / s).tolist())
    # beyond the Gram slack: the fp32 sums of the layer-norm and one-row sites, a relative 1e-3 at most
    assert (err <= slack + 1e-3 * want).all(), (s, want, slack)


@pytest.mark.parametrize("kind", ["bert", "bert_pad", "gpt"])
def test_unclipped_noiseless_full_step_is_the_plain_step(kind, monkeypatch):
    """C above every bound, z = 0: c = 1; every 2-D weight gradient is bit-identical to the plain step through
    the single-writer GEMM, and a rerun gives the same bits.  Biases, layer norms and embeddings are fixed-order
    sums of the same values the plain path adds with atomics in no fixed order: they agree within 2^-12 of the
    parameter's largest entry.  A bias sums the bf16 rows the weight GEMM reads, where the plain path sums
    the fp32 values before rounding: within 2^-8 sum_r |dz_r|."""
    _snapshot(monkeypatch)
    net, B = _net(kind)
    x, y = _inputs(kind, net, B)
    state = _state(net)
    dp = D.DPSGDStep(net.spec, B, 1e30, 0.0, 0, _word(), DEV)
    got = _grad(net, x, y, state, dp)
    assert torch.equal(got, _grad(net, x, y, state, dp))
    assert torch.equal(dp.c, torch.ones(B, device=DEV)) and int(dp.dropped) == 0
    col_abs = {r[4].data_ptr(): r[1].double().abs().sum(0) for r in dp._snap if r[0] == "lin" and r[4] is not None}
    monkeypatch.setattr(F, "_split_k", lambda *a: 1)
    plain = _grad(net, x, y, state)
    G_, P_ = net.spec.views(got), net.spec.views(plain)
    Gs = net.spec.views(state[2])
    for e in net.spec.entries:
        a, b = G_[e.name].double(), P_[e.name].double()
        if len(e.shape) == 2 and not e.name.startswith("emb."):
            assert torch.equal(a, b), e.name
        else:
            ptr = Gs[e.name].data_ptr()
            tol = 2 ** -8 * col_abs[ptr] + 1e-7 if ptr in col_abs else 2 ** -12 * b.abs().max() + 1e-7
            assert ((a - b).abs() <= tol).all(), (e.name, float((a - b).abs().max()))
    assert float(got.abs().sum()) > 0


@pytest.mark.parametrize("kind", ["bert_pad", "gpt"])
def test_clipped_full_step_against_fp64_per_example_clipping(kind, monkeypatch):
    _snapshot(monkeypatch)
    net, B = _net(kind)
    x, y = _inputs(kind, net, B, seed=4)
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
    assert (c < 1).any() and (c <= ideal * (1 + 1e-6)).all()
    ref = (g * c[:, None]).sum(0) / B
    # the realised rows are bf16(c dz): within 2^-8 + 2^-10 of the fp64 sum, relative to its norm
    rel = float((got - ref).norm() / ref.norm())
    print(kind, "relative error of the clipped step", rel)
    assert rel < 2 ** -6
    print(kind, "c / ideal", (c / ideal).tolist())
    assert float((c / ideal).min()) > 0.5


@pytest.mark.parametrize("kind", ["bert", "gpt"])
def test_single_example_contribution_is_within_the_clip(kind):
    net, _ = _net(kind)
    x, y = _inputs(kind, net, 1, seed=6)
    state = _state(net)
    unclipped = _grad(net, x, y, state, D.DPSGDStep(net.spec, 1, 1e30, 0.0, 0, _word(), DEV))
    clip = 0.25 * float(unclipped.double().norm())
    got = _grad(net, x, y, state, D.DPSGDStep(net.spec, 1, clip, 0.0, 0, _word(), DEV))
    n = float(got.double().norm())
    print(f"{kind}: B = 1 contribution {n / clip:.4f} C")
    assert 0.3 * clip < n <= clip, (n, clip)


def test_non_finite_example_is_dropped_and_the_step_stays_finite(monkeypatch):
    """A NaN in one example's rows of a layer-norm site: that example's bound is not finite, c = 0, and the
    step's gradient is finite."""
    rec = D.DPSGDStep.record_layernorm

    def poison(self, dy, x, mean, rstd, gg, gb):
        R = dy.shape[0] // self.B
        dy[2 * R + 5, 7] = float("nan")
        return rec(self, dy, x, mean, rstd, gg, gb)

    monkeypatch.setattr(D.DPSGDStep, "record_layernorm", poison)
    net, B = _net("gpt")
    x, y = _inputs("gpt", net, B, seed=8)
    state = _state(net)
    dp = D.DPSGDStep(net.spec, B, 1e30, 0.0, 0, _word(), DEV)
    got = _grad(net, x, y, state, dp)
    assert int(dp.dropped) == 1 and float(dp.c[2]) == 0.0 and torch.isfinite(got).all()
    assert float(got.abs().sum()) > 0


def test_noise_is_z_c_over_b():
    net, B = _net("gpt")
    x, y = _inputs("gpt", net, B, seed=9)
    state = _state(net)
    clip, z, seed, add = 0.5, 2.0, 0xBEEF, 2
    word = torch.tensor([17], device=DEV, dtype=torch.int32)

    def step(noise):
        master, shadow, grad = state
        grad.zero_()
        loss = net.loss(net.bind(master, shadow, grad), x, y)
        dp = D.DPSGDStep(net.spec, B, clip, noise, seed, word, DEV)
        dp.begin()
        loss.backward()
        dp.finish(grad, add)
        torch.cuda.synchronize()
        return grad.clone()

    diff = (step(z).double() - step(0.0).double()).cpu()
    want = z * clip / B * torch.from_numpy(dp_gauss(seed, 17 + add, 0, net.spec.total, DPSGD_SITE)).double()
    assert float((diff - want).abs().max()) < 1e-6 * float(want.abs().max())


# ------------------------------------------------------------------ engine rounds
def _gpt_engine(capture, rounds, shard):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import GPT
    cfg = FLConfig.for_world(1, model="gpt", batch_size=8, samples_per_client=32, learning_rate=3e-3,
                             cuda_graph=capture, dpsgd_clip=0.5, dpsgd_noise=1.0, dpsgd_seed=3,
                             dpsgd_full_model=True)
    eng = GenericFedEngine(cfg, GPT(**GPT_SMALL), shard, rank=0, world=1, device=0)
    if capture:
        eng.capture()
    for _ in range(rounds):
        eng.run_round()
    torch.cuda.synchronize()
    return eng


def test_full_gpt_rounds_replay_resume_and_ledger(tmp_path):
    from bflc_demo_b200.data.synthetic import lm_corpus_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import GPT
    from bflc_demo_b200.utils.checkpoint import load_checkpoint, save_checkpoint
    shard = lm_corpus_like(1, 32, seed=3, seq_len=128, vocab=512, only=0)[0]
    a = _gpt_engine(True, 3, shard)
    assert a.capture_error == "" and a.graph_train is not None
    b = _gpt_engine(False, 4, shard)
    assert torch.equal(a.global_master, b.global_master)
    assert a.drain_blocks() == [] and b.drain_blocks() == [] and a.host_ledger.verify_chain()
    eps, _ = b.privacy_spent_local()
    assert math.isfinite(eps) and eps > 0
    path = str(tmp_path / "full.pt")
    save_checkpoint(path, b)
    for _ in range(2):
        b.run_round()
    same = GenericFedEngine(b.cfg, GPT(**GPT_SMALL), shard, rank=0, world=1, device=0)
    load_checkpoint(path, same)
    for _ in range(2):
        same.run_round()
    torch.cuda.synchronize()
    assert torch.equal(same.global_master, b.global_master)
    assert same.drain_blocks() == [] and same.host_ledger.verify_chain()
