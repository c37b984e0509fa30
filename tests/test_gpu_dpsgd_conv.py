"""DP-SGD for LeNet-5 and the GroupNorm ResNet-18 on the H100: the convolution sites' norm paths (64 x 64
product tiles with a bias column, and the Gram form) and abs term against fp64, the deterministic split-K, the
group-norm norm and release, whole-model steps and generic-engine rounds."""
import math

import pytest
import torch

from bflc_demo_b200._native import C
from bflc_demo_b200.ops import dpsgd as D
from bflc_demo_b200.ops import gemm as G
from bflc_demo_b200.ops import nn as F
from bflc_demo_b200.protocol.oracle import DPSGD_SITE, dp_gauss

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
DEV = "cuda"


def _canaried(n):
    buf = torch.full((n + 2,), float("nan"), device=DEV)
    return buf, buf[1:-1]


def _word():
    return torch.zeros(1, device=DEV, dtype=torch.int32)


# ------------------------------------------------------------------ convolution sites
# (B, R, Cout, K, bias): LeNet conv1 / conv2, the ResNet stem, 64->64 at R 1024, 64->128 stride 2, the 1x1
# stride-2 downsample, 256->256 at R 64, 512->512 at R 16
SITES = [(3, 784, 8, 80, True), (16, 100, 16, 200, True), (3, 1024, 64, 32, False), (1, 1024, 64, 576, False),
         (3, 256, 128, 576, False), (16, 64, 256, 128, False), (3, 64, 256, 2304, False), (16, 16, 512, 4608, False)]


def _site(B, R, Cout, K, integer, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    if integer:   # sparse small integers: every tile / pair partial is an exact fp32 integer
        def ints(shape):
            v = torch.randint(-2, 3, shape, generator=g, device=DEV)
            return (v * (torch.rand(shape, generator=g, device=DEV) < 1 / 16)).to(BF)
        dz, col = ints((B * R, Cout)), ints((B * R, K))
    else:
        dz = (torch.randn(B * R, Cout, generator=g, device=DEV) * 0.1).to(BF)
        col = torch.randn(B * R, K, generator=g, device=DEV).to(BF)
    return dz, col


def _ref(dz, col, B, R, bias):
    d = dz.double().view(B, R, -1)
    p = col.double().view(B, R, -1)
    if bias:
        p = torch.cat([p, torch.ones(B, R, 1, dtype=p.dtype, device=DEV)], -1)
    V = d.transpose(1, 2) @ p
    ab = (d.norm(dim=-1) * p.norm(dim=-1)).sum(-1)
    return (V ** 2).sum((1, 2)), ab


def _run(dz, col, B, R, bias, path):
    a, K = dz.shape[1], col.shape[1]
    if path == "tiles":
        n = C().dpsgd_norm_tiles(a, K, bias) * B
        buf, out = _canaried(n)
        C().dpsgd_pe_norm(dz, col, R, out, bias=bias)
    else:
        n = C().dpsgd_gram_pairs(R, True) * B
        buf, out = _canaried(n)
        C().dpsgd_pe_gram(col, col, R, float(bias), out, p1=dz, p2=dz, mode=0)
    torch.cuda.synchronize()
    assert torch.isnan(buf[0]) and torch.isnan(buf[-1])
    return out.view(-1, B).double().sum(0), out.clone()


@pytest.mark.parametrize("site", SITES)
def test_conv_norm_paths_against_fp64(site):
    B, R, Cout, K, bias = site
    path = D.conv_norm_path(R, Cout, K + bias)
    dz, col = _site(B, R, Cout, K, integer=False)
    want, ab = _ref(dz, col, B, R, bias)
    got, raw = _run(dz, col, B, R, bias, path)
    print(site, path, "rel err", float(((got - want).abs() / want).max()))
    # fp32 accumulation: within the Gram slack kappa ab^2 (tiles: far inside it)
    kap = float(D.gram_kappa(Cout, K + bias, 64 + 16))
    assert ((got - want).abs() <= kap * ab ** 2 + 1e-5 * want).all(), (got, want)
    _, again = _run(dz, col, B, R, bias, path)
    assert torch.equal(raw, again)
    expected = {784: "tiles", 100: "tiles", 1024: "tiles", 256: "tiles", 64: "gram", 16: "gram"}[R]
    assert path == expected


@pytest.mark.parametrize("site", [SITES[0], SITES[1], SITES[3], SITES[7]])
def test_conv_norm_paths_exact_on_integers(site):
    B, R, Cout, K, bias = site
    dz, col = _site(B, R, Cout, K, integer=True, seed=1)
    want, _ = _ref(dz, col, B, R, bias)
    assert float(want.max()) < 2 ** 24
    for path in ("tiles",) + (("gram",) if R <= 512 else ()):
        got, _ = _run(dz, col, B, R, bias, path)
        assert torch.equal(got, want), (path, got, want)


@pytest.mark.parametrize("B, R, K, bias", [(3, 784, 80, True), (2, 1024, 576, False), (16, 100, 200, True)])
def test_patch_abs_term_against_fp64(B, R, K, bias):
    dz, col = _site(B, R, 16, K, integer=False, seed=2)
    _, want = _ref(dz, col, B, R, bias)
    buf, ab = _canaried(B)
    C().dpsgd_pe_rows(dz, col, R, float(bias), None, ab)
    torch.cuda.synchronize()
    assert torch.isnan(buf[0]) and torch.isnan(buf[-1])
    torch.testing.assert_close(ab.double(), want, rtol=1e-5, atol=0)
    again = torch.empty_like(ab)
    C().dpsgd_pe_rows(dz, col, R, float(bias), None, again)
    assert torch.equal(ab, again)


def _conv_ints(shape, g, density=1 / 16):
    v = torch.randint(-2, 3, shape, generator=g, device=DEV)
    return (v * (torch.rand(shape, generator=g, device=DEV) < density)).to(BF)


# implicit-eligible sites: 64->64 at R 1024 (stage 1), 64->128 stride 2 (R 256), the 1x1 stride-2 downsample
IMPLICIT = [(1, 64, 32, 64, 3, 1, 1), (3, 64, 32, 64, 3, 1, 1), (3, 64, 32, 128, 3, 2, 1), (3, 64, 32, 128, 1, 2, 0)]


@pytest.mark.parametrize("B, Cin, H, Cout, k, stride, pad", IMPLICIT)
def test_both_tile_paths_agree_on_an_implicit_site(B, Cin, H, Cout, k, stride, pad):
    """The implicit weight-gradient GEMM's per-example mode (one K group per example, 128 x 64 tiles squared
    in its epilogue) and im2col + k_pe_norm (64 x 64 tiles) against fp64: exact on sparse integer fixtures,
    with NaN canaries and bit-identical reruns; the patch abs term from x against the patch rows."""
    g = torch.Generator(device=DEV).manual_seed(11)
    OH = (H + 2 * pad - k) // stride + 1
    R, K = OH * OH, k * k * Cin
    x = _conv_ints((B, H, H, Cin), g)
    dz = _conv_ints((B * R, Cout), g)
    col = torch.empty(B * R, K, device=DEV, dtype=BF)
    C().im2col(x, col, B, Cin, H, H, k, k, stride, pad, OH, OH)
    want, ab_want = _ref(dz, col, B, R, False)
    assert float(want.max()) < 2 ** 24
    n = C().conv_dw_norm_tiles(Cout, K) * B
    buf, out = _canaried(n)
    C().conv_dw_groups(x, dz, out, B, H, H, Cin, OH, OH, k, k, stride, pad, B, True)
    torch.cuda.synchronize()
    assert torch.isnan(buf[0]) and torch.isnan(buf[-1])
    got = out.view(-1, B).double().sum(0)
    assert torch.equal(got, want), (got, want)
    again = torch.empty_like(out)
    C().conv_dw_groups(x, dz, again, B, H, H, Cin, OH, OH, k, k, stride, pad, B, True)
    assert torch.equal(out, again)
    tiles, _ = _run(dz, col, B, R, False, "tiles")
    assert torch.equal(tiles, got)
    # random operands: both paths within fp32 accumulation of fp64
    xr = torch.randn(B, H, H, Cin, generator=g, device=DEV).to(BF)
    dzr = (torch.randn(B * R, Cout, generator=g, device=DEV) * 0.1).to(BF)
    C().im2col(xr, col, B, Cin, H, H, k, k, stride, pad, OH, OH)
    want, ab_want = _ref(dzr, col, B, R, False)
    C().conv_dw_groups(xr, dzr, out, B, H, H, Cin, OH, OH, k, k, stride, pad, B, True)
    torch.testing.assert_close(out.view(-1, B).double().sum(0), want, rtol=2e-5, atol=0)
    ab = torch.empty(B, device=DEV)
    C().dpsgd_patch_rows(dzr, xr, B, H, H, Cin, OH, OH, k, k, stride, pad, 0.0, ab)
    torch.testing.assert_close(ab.double(), ab_want, rtol=1e-5, atol=0)


@pytest.mark.parametrize("B, Cin, H, Cout, k, stride, pad", IMPLICIT + [(64, 64, 4, 64, 3, 1, 1)])
def test_implicit_release_by_k_groups(B, Cin, H, Cout, k, stride, pad):
    """conv_dw_fixed_split: whole-example K groups stored into slices and added in order; exact on integer
    fixtures, bit-identical on rerun, and equal to the GEMM over the patches."""
    g = torch.Generator(device=DEV).manual_seed(12)
    OH = (H + 2 * pad - k) // stride + 1
    R, K = OH * OH, k * k * Cin
    x = _conv_ints((B, H, H, Cin), g, 1 / 4)
    dz = _conv_ints((B * R, Cout), g, 1 / 4)
    geom = (B, Cin, H, H, k, k, stride, pad, OH, OH)
    gw = torch.full((Cout, K), 0.5, device=DEV)
    G.conv_dw_fixed_split(x, dz, gw, geom, B)
    again = torch.full((Cout, K), 0.5, device=DEV)
    G.conv_dw_fixed_split(x, dz, again, geom, B)
    col = torch.empty(B * R, K, device=DEV, dtype=BF)
    C().im2col(x, col, B, Cin, H, H, k, k, stride, pad, OH, OH)
    torch.cuda.synchronize()
    assert torch.equal(gw, again)
    assert torch.equal(gw.double(), 0.5 + dz.double().t() @ col.double())


def test_k_group_gemm_refusals():
    g = torch.Generator(device=DEV).manual_seed(13)
    x = _conv_ints((3, 4, 4, 64), g)
    dz = _conv_ints((3 * 16, 64), g)
    out = torch.empty(C().conv_dw_norm_tiles(64, 576) * 3, device=DEV)
    with pytest.raises(RuntimeError, match="multiple of 64 pixels"):    # R 16: a 64-pixel box spans examples
        C().conv_dw_groups(x, dz, out, 3, 4, 4, 64, 4, 4, 3, 3, 1, 1, 3, True)
    with pytest.raises(RuntimeError, match="multiple of 64 pixels"):    # groups must divide the examples
        C().conv_dw_groups(x, dz, out, 3, 4, 4, 64, 4, 4, 3, 3, 1, 1, 2, True)
    with pytest.raises(ValueError, match="multiple of 64 pixels"):
        G.conv_dw_fixed_split(x, dz, torch.zeros(64, 576, device=DEV), (3, 64, 4, 4, 3, 3, 1, 1, 4, 4), 3)


@pytest.mark.parametrize("Cin, H, Cout, stride", [(64, 32, 64, 1), (64, 32, 128, 2)])
def test_implicit_and_im2col_layers_agree(Cin, H, Cout, stride, monkeypatch):
    """The same convolution through the implicit-GEMM layer (per-example GEMM norms, patch norms from x,
    K-group release) and the im2col layer (patches): on integer fixtures the per-example norms and the clipped
    release agree exactly, the abs terms to fp32 rounding."""
    g = torch.Generator(device=DEV).manual_seed(5)
    B = 3
    x = _conv_ints((B, H, H, Cin), g)
    w = _conv_ints((Cout, 9 * Cin), g)
    OH = (H + 2 - 3) // stride + 1
    dy = _conv_ints((B, OH, OH, Cout), g)
    outs = []
    for implicit in (True, False):
        monkeypatch.setattr(F, "_IMPLICIT", implicit)
        assert F.conv_is_implicit(H, H, Cin, 3, 3, stride, 1, 9 * Cin) == implicit
        gw = torch.zeros(Cout, 9 * Cin, device=DEV)
        dp = D.DPSGDStep(_spec([(Cout, 9 * Cin)]), B, 1e30, 0.0, 0, _word(), DEV, conv=True)
        xi = x.clone().requires_grad_(True)
        y = F.conv2d(xi, w, None, gw, None, 3, 3, stride, 1)
        dp.begin()
        y.backward(dy)
        kinds = [r[0] for r in dp._records]
        dp.finish(gw, 0)
        torch.cuda.synchronize()
        assert kinds == (["convx"] if implicit else ["conv"])
        outs.append((dp.sq[:dp._n_sq].double().sum(0), dp.ab[:dp._n_ab].clone(), gw.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][2], outs[1][2])
    torch.testing.assert_close(outs[0][1], outs[1][1], rtol=1e-6, atol=0)
    assert float(outs[0][2].abs().sum()) > 0


def _spec(shapes):
    from bflc_demo_b200.models.flat import ParamSpec
    return ParamSpec([(f"p{i}", s) for i, s in enumerate(shapes)])


# ------------------------------------------------------------------ deterministic split-K
@pytest.mark.parametrize("B, R, Cout, K", [(64, 1024, 64, 576), (128, 784, 8, 80), (4, 16, 512, 4608)])
def test_fixed_split_dw_is_reproducible_and_within_the_fp32_bound(B, R, Cout, K):
    dz, col = _site(B, R, Cout, K, integer=False, seed=3)
    s = G.fixed_splits(B * R, Cout, K, B)
    gw = torch.full((Cout, K), 0.25, device=DEV)
    G.gemm_dw_fixed_split(dz, col, gw, s)
    again = torch.full((Cout, K), 0.25, device=DEV)
    G.gemm_dw_fixed_split(dz, col, again, s)
    torch.cuda.synchronize()
    assert torch.equal(gw, again)
    want = 0.25 + dz.double().t() @ col.double()
    bound = (B * R + s + 1) * 2.0 ** -23 * (dz.double().abs().t() @ col.double().abs() + 0.25)
    assert ((gw.double() - want).abs() <= bound).all()
    print((B, R, Cout, K), "splits", s)


def test_fixed_split_dw_refusals():
    dz, col = _site(3, 16, 8, 16, integer=False)
    gw = torch.zeros(8, 16, device=DEV)
    with pytest.raises(ValueError, match="do not divide"):
        G.gemm_dw_fixed_split(dz, col, gw, 5)
    with pytest.raises(ValueError, match="contiguous fp32"):
        G.gemm_dw_fixed_split(dz, col, gw.to(BF), 3)
    with pytest.raises(ValueError, match="contiguous fp32"):
        G.gemm_dw_fixed_split(dz, col, torch.zeros(16, 8, device=DEV).t(), 3)
    with pytest.raises(ValueError, match="bf16"):
        G.gemm_dw_fixed_split(dz.float(), col, gw, 3)


# ------------------------------------------------------------------ group norms
def test_gn_norm_and_release_exact_against_a_fixed_order_model():
    g = torch.Generator(device=DEV).manual_seed(7)
    N, Cc = 5, 96
    pg = torch.randn(N, Cc, generator=g, device=DEV)
    pb = torch.randn(N, Cc, generator=g, device=DEV)
    sq = torch.empty(N, device=DEV)
    C().dpsgd_pe_gn(pg, pb, sq)
    torch.testing.assert_close(sq.double(), (pg.double() ** 2 + pb.double() ** 2).sum(1), rtol=1e-6, atol=0)
    cf = torch.tensor([1.0, 0.0, 0.5, 0.3, 1.0], device=DEV)
    pg[1, 3] = float("nan")                      # a dropped example's partials may be non-finite
    gg, gb = torch.full((Cc,), 0.5, device=DEV), torch.zeros(Cc, device=DEV)
    C().groupnorm_param(pg, pb, gg, gb, cf=cf)
    # model: a = 0; for each n with c_n != 0, a = fl(a + fl(c_n pg)), then g += a, all in fp32
    a = torch.zeros(Cc, device=DEV)
    b = torch.zeros(Cc, device=DEV)
    for n in range(N):
        if float(cf[n]) != 0.0:
            a = a + cf[n] * pg[n]
            b = b + cf[n] * pb[n]
    torch.cuda.synchronize()
    assert torch.equal(gg, 0.5 + a) and torch.equal(gb, b)
    # no factor: today's plain sums, the bits groupnorm_bwd adds
    pg[1, 3] = 1.0
    gg2, gb2 = torch.zeros(Cc, device=DEV), torch.zeros(Cc, device=DEV)
    C().groupnorm_param(pg, pb, gg2, gb2)
    a = torch.zeros(Cc, device=DEV)
    for n in range(N):
        a = a + pg[n]
    assert torch.equal(gg2, a)


# ------------------------------------------------------------------ whole models
@pytest.fixture(autouse=True)
def _deterministic_convolutions():
    """As GenericFedEngine sets it for DP-SGD: no split-K atomics in the convolutions' forward / input gradient."""
    prev = F.set_deterministic(True)
    yield
    F.set_deterministic(prev)


def _net(kind):
    from bflc_demo_b200.models.nets import LeNet5, ResNet18
    return (LeNet5(), 8) if kind == "lenet5" else (ResNet18(norm="group"), 3)


def _inputs(net, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (B, 3, 32, 32), generator=g, dtype=torch.uint8)
    return net.preprocess(x.to(DEV)), torch.randint(0, 10, (B,), generator=g).to(DEV, torch.int32)


def _state(net, seed=3):
    master = torch.zeros(net.spec.total, device=DEV)
    net.init_(master, seed=seed)
    return master, master.to(BF), torch.zeros(net.spec.total, device=DEV)


def _grad(net, x, y, state, dp=None):
    master, shadow, grad = state
    grad.zero_()
    loss = net.loss(net.bind(master, shadow, grad), x, y)
    if dp is None:
        loss.backward()
    else:
        dp.begin()
        loss.backward()
        dp.finish(grad, 0)
    torch.cuda.synchronize()
    return grad.clone()


def _snapshot(monkeypatch):
    fin = D.DPSGDStep.finish

    def spy(self, grad, add):
        self._snap = list(self._records)
        return fin(self, grad, add)

    monkeypatch.setattr(D.DPSGDStep, "finish", spy)


def _linear_view(rec):
    """A linear or convolution record as (dz, operand, gw, gb, R); an implicit-GEMM convolution's patches are
    built here (the step never forms them)."""
    if rec[0] == "convx":
        _, dz, x, geom, gw, R, _ = rec
        N, Cin, H, W, kh, kw, stride, pad, OH, OW = geom
        col = torch.empty(dz.shape[0], kh * kw * Cin, device=DEV, dtype=BF)
        C().im2col(x, col, N, Cin, H, W, kh, kw, stride, pad, OH, OW)
        return dz, col, gw, None, R
    _, dz, op, gw, gb, R, _ = rec
    return dz, op, gw, gb, R


def _per_example_fp64(dp, net, state, B):
    """Each example's gradient over the flat vector in fp64 from the recorded sites (dz_n^T (x_n, 1) of linear
    and convolution sites, the group norms' partials), times B (the rows are of the batch-mean loss)."""
    out = torch.zeros(B, net.spec.total, dtype=torch.float64, device=DEV)
    base = state[2].data_ptr()

    def put(n, g, val):
        off = (g.data_ptr() - base) // 4
        out[n, off:off + g.numel()].view(g.shape).add_(val)

    for rec in dp._snap:
        lin = _linear_view(rec) if rec[0] in ("lin", "conv", "convx") else None
        for n in range(B):
            if lin is not None:
                dz, op, gw, gb, R = lin
                sl = slice(n * R, (n + 1) * R)
                if gw is not None:
                    put(n, gw, dz[sl].double().t() @ op[sl].double())
                if gb is not None:
                    put(n, gb, dz[sl].double().sum(0))
            else:
                _, pg, pb, gg, gb = rec
                if gg is not None:
                    put(n, gg, pg[n].double())
                if gb is not None:
                    put(n, gb, pb[n].double())
    return out * B


@pytest.mark.parametrize("kind", ["lenet5", "resnet18"])
def test_per_example_norms_match_fp64_over_the_whole_vector(kind, monkeypatch):
    _snapshot(monkeypatch)
    net, B = _net(kind)
    x, y = _inputs(net, B)
    state = _state(net)
    dp = D.DPSGDStep(net.spec, B, 1e30, 0.0, 0, _word(), DEV, conv=True)
    _grad(net, x, y, state, dp)
    kinds = {r[0] for r in dp._snap}
    assert "conv" in kinds and (kind == "lenet5" or {"gn", "convx"} <= kinds)
    g = _per_example_fp64(dp, net, state, B)
    want = g.pow(2).sum(1) / B ** 2
    s = dp.sq[:dp._n_sq].double().sum(0)
    slack = (dp.kap[:dp._n_ab].double()[:, None] * dp.ab[:dp._n_ab].double() ** 2).sum(0)
    err = (s - want).abs()
    print(kind, "rel err", (err / want).tolist(), "slack / s", (slack / s).tolist())
    assert (err <= slack + 1e-4 * want).all(), (s, want, slack)


@pytest.mark.parametrize("kind", ["lenet5", "resnet18"])
def test_unclipped_noiseless_step_is_the_plain_step(kind, monkeypatch):
    """C above every bound, z = 0: c = 1, nothing dropped, and a rerun gives the same bits.  Convolution and
    linear weights agree with the plain step within the plain path's split-K reordering (fp32 atomics, no
    fixed order): both are within (rows + 64) 2^-24 |dz|^T |x| of the exact sum.  Group norms: the plain path
    adds the same partials in the same order (c = 1 multiplies exactly), so they are equal.  Biases sum the bf16 rows the GEMM reads: within 2^-8
    of sum_r |dz_r|."""
    _snapshot(monkeypatch)
    net, B = _net(kind)
    x, y = _inputs(net, B, seed=2)
    state = _state(net)
    dp = D.DPSGDStep(net.spec, B, 1e30, 0.0, 0, _word(), DEV, conv=True)
    got = _grad(net, x, y, state, dp)
    assert torch.equal(got, _grad(net, x, y, state, dp))
    assert torch.equal(dp.c, torch.ones(B, device=DEV)) and int(dp.dropped) == 0
    lins = [_linear_view(r) for r in dp._snap if r[0] in ("lin", "conv", "convx")]
    col_abs = {gb.data_ptr(): dz.double().abs().sum(0) for dz, _, _, gb, _ in lins if gb is not None}
    w_abs = {gw.data_ptr(): (dz.shape[0] + 64) * 2.0 ** -23 * (dz.double().abs().t() @ op.double().abs())
             for dz, op, gw, _, _ in lins if gw is not None}
    plain = _grad(net, x, y, state)
    G_, P_, Gs = net.spec.views(got), net.spec.views(plain), net.spec.views(state[2])
    for e in net.spec.entries:
        a, b = G_[e.name].double(), P_[e.name].double()
        ptr = Gs[e.name].data_ptr()
        if len(e.shape) == 2:
            tol = w_abs[ptr] + 1e-12
        elif ptr in col_abs:
            tol = 2 ** -8 * col_abs[ptr] + 1e-7
        else:
            assert torch.equal(a, b), e.name
            continue
        assert ((a - b).abs() <= tol).all(), (e.name, float((a - b).abs().max()))
    assert float(got.abs().sum()) > 0


@pytest.mark.parametrize("kind", ["lenet5", "resnet18"])
def test_clipped_step_against_fp64_per_example_clipping(kind, monkeypatch):
    _snapshot(monkeypatch)
    net, B = _net(kind)
    x, y = _inputs(net, B, seed=4)
    state = _state(net)
    probe = D.DPSGDStep(net.spec, B, 1e30, 0.0, 0, _word(), DEV, conv=True)
    _grad(net, x, y, state, probe)
    g = _per_example_fp64(probe, net, state, B)
    norms = g.norm(dim=1)
    clip = float(norms.median())
    dp = D.DPSGDStep(net.spec, B, clip, 0.0, 0, _word(), DEV, conv=True)
    got = _grad(net, x, y, state, dp).double()
    c = dp.c.double()
    ideal = (clip / norms).clamp(max=1)
    assert (c < 1).any() and (c <= ideal * (1 + 1e-6)).all()
    ref = (g * c[:, None]).sum(0) / B
    rel = float((got - ref).norm() / ref.norm())
    print(kind, "relative error of the clipped step", rel, "c / ideal", (c / ideal).tolist())
    assert rel < 2 ** -6 and float((c / ideal).min()) > 0.5


@pytest.mark.parametrize("kind", ["lenet5", "resnet18"])
def test_single_example_contribution_is_within_the_clip(kind):
    net, _ = _net(kind)
    x, y = _inputs(net, 1, seed=6)
    state = _state(net)
    unclipped = _grad(net, x, y, state, D.DPSGDStep(net.spec, 1, 1e30, 0.0, 0, _word(), DEV, conv=True))
    clip = 0.25 * float(unclipped.double().norm())
    got = _grad(net, x, y, state, D.DPSGDStep(net.spec, 1, clip, 0.0, 0, _word(), DEV, conv=True))
    n = float(got.double().norm())
    print(f"{kind}: B = 1 contribution {n / clip:.4f} C")
    assert 0.3 * clip < n <= clip, (n, clip)


@pytest.mark.parametrize("kind", ["lenet5", "resnet18"])
def test_non_finite_example_is_dropped_and_the_step_stays_finite(kind):
    net, B = _net(kind)
    x, y = _inputs(net, B, seed=8)
    x[1, 5, 5, 0] = float("nan")
    state = _state(net)
    dp = D.DPSGDStep(net.spec, B, 1e30, 0.0, 0, _word(), DEV, conv=True)
    got = _grad(net, x, y, state, dp)
    assert int(dp.dropped) == 1 and float(dp.c[1]) == 0.0 and torch.isfinite(got).all()
    assert float(got.abs().sum()) > 0


def test_noise_is_z_c_over_b():
    net, B = _net("lenet5")
    x, y = _inputs(net, B, seed=9)
    state = _state(net)
    clip, z, seed, add = 0.5, 2.0, 0xBEEF, 2
    word = torch.tensor([17], device=DEV, dtype=torch.int32)

    def step(noise):
        master, shadow, grad = state
        grad.zero_()
        loss = net.loss(net.bind(master, shadow, grad), x, y)
        dp = D.DPSGDStep(net.spec, B, clip, noise, seed, word, DEV, conv=True)
        dp.begin()
        loss.backward()
        dp.finish(grad, add)
        torch.cuda.synchronize()
        return grad.clone()

    diff = (step(z).double() - step(0.0).double()).cpu()
    want = z * clip / B * torch.from_numpy(dp_gauss(seed, 17 + add, 0, net.spec.total, DPSGD_SITE)).double()
    assert float((diff - want).abs().max()) < 1e-6 * float(want.abs().max())


# ------------------------------------------------------------------ engine rounds
def _engine(kind, capture, shard):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import LeNet5, ResNet18
    norm = dict(resnet_norm="group") if kind == "resnet18" else {}
    cfg = FLConfig.for_world(1, model=kind, batch_size=8, samples_per_client=32, learning_rate=0.01,
                             cuda_graph=capture, dpsgd_clip=1.0, dpsgd_noise=1.0, dpsgd_seed=3, dpsgd_conv=True,
                             **norm)
    net = LeNet5() if kind == "lenet5" else ResNet18(norm="group")
    eng = GenericFedEngine(cfg, net, shard, rank=0, world=1, device=0)
    if capture:
        eng.capture()
    return eng, net


@pytest.mark.parametrize("kind", ["lenet5", "resnet18"])
def test_rounds_replay_resume_ledger_and_epsilon(kind, tmp_path):
    from bflc_demo_b200.data.synthetic import cifar_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.utils.checkpoint import load_checkpoint, save_checkpoint
    shard = cifar_like(1, 32, seed=3, alpha=0.0)[0]
    a, _ = _engine(kind, True, shard)           # one eager round, then the graph
    assert a.capture_error == "" and a.graph_train is not None
    for _ in range(2):
        a.run_round()
    b, net = _engine(kind, False, shard)
    for _ in range(3):
        b.run_round()
    torch.cuda.synchronize()
    assert torch.equal(a.global_master, b.global_master)
    assert a.drain_blocks() == [] and b.drain_blocks() == [] and a.host_ledger.verify_chain()
    eps, _ = b.privacy_spent_local()
    assert math.isfinite(eps) and eps > 0
    path = str(tmp_path / f"{kind}.pt")
    save_checkpoint(path, b)
    for _ in range(2):
        b.run_round()
    same = GenericFedEngine(b.cfg, type(net)() if kind == "lenet5" else type(net)(norm="group"), shard,
                            rank=0, world=1, device=0)
    load_checkpoint(path, same)
    for _ in range(2):
        same.run_round()
    torch.cuda.synchronize()
    assert torch.equal(same.global_master, b.global_master)
    assert same.drain_blocks() == [] and same.host_ledger.verify_chain()
    assert int(b.dpsgd.dropped.item()) == 0
