"""Conformance of the layers the LeNet-5, ResNet-18 and BERT configs run on top of the GEMMs: both
convolution paths (``ops.nn.ConvImplicitFn``: ``ConvView`` in ``csrc/kernels/gemm_sm100.cu``;
``ops.nn.Conv2dFn``: im2col + GEMM + col2im) and every layer of ``csrc/kernels/nn_kernels.cu``,
against plain float64 references defined here.

Two kinds of comparison, as in ``test_gpu_gemm_conformance.py``:

* exact -- operands are small integers chosen per case so that every fp32 sum is exact and every
  value a kernel path stores in bf16 is representable (``test_conv_operands_are_exact`` checks
  this from the operands on the CPU).  An fp32 result must equal the fp64 reference, a bf16 result
  the reference rounded once.
* bound -- elementwise ``|out - ref| <= derived slack + half an ulp of out's type``, the slack
  derived from the kernel's accumulation (its fp32 reduction depth, ``rsqrtf`` / ``__expf``).

The references follow the kernels' conventions where they differ from torch's: channels-last
weights ``[Cout][kh][kw][Cin]`` padded to ``Kp`` columns, max pool keeping the first maximum in
window scan order (a window of -inf only gives index -1).  Tests marked ``gpu`` need an H100; the
reference self-check and the exactness guard run anywhere.
"""
import math
from typing import NamedTuple

import pytest
import torch

from bflc_demo_b200._native import C

gpu = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U32 = 2.0 ** -24                                   # fp32 unit roundoff
HALF_ULP = {F32: 2.0 ** -24, BF16: 2.0 ** -8}      # relative, normal range
FLOOR = {F32: 2.0 ** -126, BF16: 2.0 ** -126}
ACT_NONE, ACT_RELU, ACT_GELU = 0, 1, 2
BF16_INT = 256                                     # every integer of magnitude <= 256 is a bf16 value
F32_INT = 2 ** 24


# ------------------------------------------------------------------------------------ helpers
def gen(seed):
    return torch.Generator().manual_seed(seed)


def ints(g, *shape, r=1, density=1.0):
    """float64 CPU tensor of integers in [-r, r]; each entry kept with probability ``density``."""
    v = torch.randint(-r, r + 1, shape, generator=g).double()
    if density < 1.0:
        v = v * (torch.rand(shape, generator=g, dtype=F64) < density)
    return v


def exact_violations(out, ref):
    """Elements of ``out`` that differ from ``ref`` (float64, exact in fp32) rounded once to
    ``out``'s type.  Raises if the reference itself is not exact in fp32."""
    ref = ref.to(out.device)
    r32 = ref.to(F32)
    assert torch.equal(r32.double(), ref), "exact reference needs fp32-exact values"
    want = r32.to(out.dtype).float() if out.dtype != F32 else r32
    return out.float() != want


def bound_violations(out, ref, slack):
    """Elements with ``|out - ref| > slack + half an ulp of out's type at |ref|``; ``slack`` is a
    float64 tensor or number (the derived error of the kernel's fp32 arithmetic)."""
    ref = ref.to(out.device)
    if torch.is_tensor(slack):
        slack = slack.to(out.device)
    tol = slack + HALF_ULP[out.dtype] * ref.abs() * (1 + 2.0 ** -10) + FLOOR[out.dtype]
    o = out.double()
    return ~torch.isfinite(o) | ((o - ref).abs() > tol)


def _report(bad, out, ref, what):
    n = int(bad.sum())
    if n:
        idx = tuple(int(i) for i in bad.nonzero()[0])
        got, want = float(out[idx]), float(ref.to(out.device)[idx])
        raise AssertionError(f"{what}: {n} of {bad.numel()} elements wrong, first at {idx}: "
                             f"{got!r} against {want!r}")


def assert_exact(out, ref, what):
    _report(exact_violations(out, ref), out, ref, what)


def assert_bound(out, ref, slack, what):
    _report(bound_violations(out, ref, slack), out, ref, what)


def launches():
    return C().launch_count()


def rows_per_lane(rows, gy):
    """Sequential fp32 additions of one lane of the 32-channel x 8-row-lane reductions
    (``k_bn_stats``, ``k_bn_bwd_reduce``, ``k_act_bwd_colsum``) plus the 8-lane combine and the
    ``gy`` atomics into the target: the depth of every partial sum."""
    return -(-rows // (8 * gy)) + 8 + gy


def grid_y(rows, cap):
    return max(1, min(cap, rows // 64))


# ---------------------------------------------------------------- float64 layer references
def out_hw(H, W, k, s, p):
    return (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1


def taps(Wm, k, cin):
    """[Cout, Kp] (column (kh*k + kw)*Cin + c, pad columns past k*k*Cin) -> [k, k, Cout, Cin]."""
    return Wm[:, :k * k * cin].reshape(Wm.shape[0], k, k, cin).permute(1, 2, 0, 3)


def conv_ref(X, Wm, k, s, p, drop_border=False):
    """y[n, oh, ow, :] = sum over taps of x[n, oh*s - p + a, ow*s - p + b, :] @ w[:, a, b, :]^T.
    ``drop_border`` (self-check perturbation): the first output row loses its last tap row, the
    one that reads real input rows there."""
    N, H, W, cin = X.shape
    OH, OW = out_hw(H, W, k, s, p)
    Xp = X.new_zeros(N, H + 2 * p, W + 2 * p, cin)
    Xp[:, p:p + H, p:p + W] = X
    T = taps(Wm, k, cin)
    y = X.new_zeros(N, OH, OW, Wm.shape[0])
    for a in range(k):
        for b in range(k):
            part = Xp[:, a:a + s * (OH - 1) + 1:s, b:b + s * (OW - 1) + 1:s] @ T[a, b].t()
            if drop_border and a == k - 1:
                part[:, 0] = 0
            y += part
    return y


def conv_dx_ref(dZ, Wm, H, W, cin, k, s, p):
    """Input gradient by scattering each tap's dz @ w back to the pixels it read."""
    N, OH, OW, _ = dZ.shape
    T = taps(Wm, k, cin)
    dXp = dZ.new_zeros(N, H + 2 * p, W + 2 * p, cin)
    for a in range(k):
        for b in range(k):
            dXp[:, a:a + s * (OH - 1) + 1:s, b:b + s * (OW - 1) + 1:s] += dZ @ T[a, b]
    return dXp[:, p:p + H, p:p + W]


def conv_dx_upsample_ref(dZ, Wm, H, W, cin, k, s, p, shift=0):
    """The same input gradient the way the implicit path forms it for stride s: dz zero-stuffed on
    the input grid (``up[s*oh + shift, s*ow] = dz[oh, ow]``), then a stride-1 convolution with
    the taps flipped.  ``shift`` = 1 is a self-check perturbation."""
    N, OH, OW, cout = dZ.shape
    up = dZ.new_zeros(N, H + s, W, cout)
    up[:, shift:shift + s * OH:s, 0:s * OW:s] = dZ
    up = up[:, :H]
    T = taps(Wm, k, cin)
    U = dZ.new_zeros(N, H + 2 * k, W + 2 * k, cout)
    U[:, k:k + H, k:k + W] = up
    dx = dZ.new_zeros(N, H, W, cin)
    for a in range(k):
        for b in range(k):
            dx += U[:, k + p - a:k + p - a + H, k + p - b:k + p - b + W] @ T[a, b]
    return dx


def conv_dw_ref(X, dZ, k, s, p, Kp):
    N, H, W, cin = X.shape
    OH, OW = out_hw(H, W, k, s, p)
    cout = dZ.shape[-1]
    Xp = X.new_zeros(N, H + 2 * p, W + 2 * p, cin)
    Xp[:, p:p + H, p:p + W] = X
    gw = X.new_zeros(cout, Kp)
    dz = dZ.reshape(-1, cout)
    for a in range(k):
        for b in range(k):
            t = a * k + b
            patch = Xp[:, a:a + s * (OH - 1) + 1:s, b:b + s * (OW - 1) + 1:s].reshape(-1, cin)
            gw[:, t * cin:(t + 1) * cin] = dz.t() @ patch
    return gw


def im2col_ref(X, k, s, p):
    """[N*OH*OW, k*k*C], column (a*k + b)*C + c."""
    N, H, W, cin = X.shape
    OH, OW = out_hw(H, W, k, s, p)
    Xp = X.new_zeros(N, H + 2 * p, W + 2 * p, cin)
    Xp[:, p:p + H, p:p + W] = X
    cols = [Xp[:, a:a + s * (OH - 1) + 1:s, b:b + s * (OW - 1) + 1:s] for a in range(k) for b in range(k)]
    return torch.cat(cols, -1).reshape(N * OH * OW, k * k * cin)


def col2im_ref(col, N, H, W, cin, k, s, p):
    OH, OW = out_hw(H, W, k, s, p)
    c = col[:, :k * k * cin].reshape(N, OH, OW, k, k, cin)
    dXp = col.new_zeros(N, H + 2 * p, W + 2 * p, cin)
    for a in range(k):
        for b in range(k):
            dXp[:, a:a + s * (OH - 1) + 1:s, b:b + s * (OW - 1) + 1:s] += c[:, :, :, a, b]
    return dXp[:, p:p + H, p:p + W]


def gelu_ref(z):
    return 0.5 * z * (1 + torch.special.erf(z / 2 ** 0.5))


def gelu_grad_ref(z):
    return 0.5 * (1 + torch.special.erf(z / 2 ** 0.5)) + z * torch.exp(-0.5 * z * z) / (2 * math.pi) ** 0.5


def maxpool_ref(X, k, s, p, tie="first"):
    """-> (y, idx): first strict maximum in window scan order (rows, then columns); idx is the
    offset (ih*W + iw)*C + c inside the sample, -1 when every tap is -inf or padding.
    ``tie="last"`` (self-check perturbation) keeps the last maximum instead."""
    N, H, W, Cc = X.shape
    OH, OW = out_hw(H, W, k, s, p)
    best = torch.full((N, OH, OW, Cc), -math.inf, dtype=F64)
    bi = torch.full((N, OH, OW, Cc), -1, dtype=torch.int64)
    cidx = torch.arange(Cc)
    for a in range(k):
        for b in range(k):
            for oh in range(OH):
                ih = oh * s - p + a
                if not 0 <= ih < H:
                    continue
                for ow in range(OW):
                    iw = ow * s - p + b
                    if not 0 <= iw < W:
                        continue
                    v = X[:, ih, iw, :].double().cpu()
                    take = (v > best[:, oh, ow]) if tie == "first" else ((v >= best[:, oh, ow]) & (v > -math.inf))
                    best[:, oh, ow] = torch.where(take, v, best[:, oh, ow])
                    bi[:, oh, ow] = torch.where(take, (ih * W + iw) * Cc + cidx, bi[:, oh, ow])
    return best, bi


def maxpool_dx_ref(dY, idx, H, W, Cc):
    N = dY.shape[0]
    dx = torch.zeros(N, H * W * Cc, dtype=F64)
    d, i = dY.double().cpu().reshape(N, -1), idx.cpu().reshape(N, -1)
    keep = i >= 0
    for n in range(N):
        dx[n].index_add_(0, i[n][keep[n]], d[n][keep[n]])
    return dx.view(N, H, W, Cc)


class BNStats(NamedTuple):
    mean: torch.Tensor
    var: torch.Tensor
    rstd: torch.Tensor
    mean_tol: torch.Tensor          # absolute
    rstd_tol: torch.Tensor          # relative


def bn_stats_ref(x, eps=1e-5, ddof=0):
    """Per-channel mean, biased variance and rstd of x [rows, C] (float64), with the error a
    correct fp32 kernel may make: sums of x - x[0, c] (pivot: the first row) accumulated to the
    depth of the 32 x 8 lane grid, then ``mean = pivot + S1/rows``, ``var = S2/rows - (S1/rows)^2``
    and ``rsqrtf``.  The rstd bound is capped at 2^-14 relative.  ``ddof`` = 1 is a self-check
    perturbation (variance over rows - 1)."""
    rows = x.shape[0]
    depth = rows_per_lane(rows, grid_y(rows, 64))
    mean = x.mean(0)
    var = ((x - mean) ** 2).sum(0) / (rows - ddof) if rows > ddof else torch.zeros_like(mean)
    rstd = 1.0 / torch.sqrt(var + eps)
    d = x - x[0]
    s1 = d.abs().sum(0) / rows
    s2 = (d * d).sum(0) / rows
    m1 = (d.sum(0) / rows).abs()
    mean_tol = 2 * (depth * U32 * s1 + 2 * U32 * mean.abs())
    var_err = 2 * ((depth + 1) * U32 * s2 + 2 * m1 * depth * U32 * s1 + 4 * U32 * (s2 + m1 * m1) + U32 * eps)
    rstd_tol = torch.clamp(0.5 * var_err / (var + eps) + 4 * U32, max=2.0 ** -14)
    return BNStats(mean, var, rstd, mean_tol, rstd_tol)


def ln_stats_ref(x, eps=1e-12, cols=None):
    """Per-row mean and rstd of x [rows, C] (float64) over the first ``cols`` columns (all by
    default; C - 1 is a self-check perturbation), with the error of ``k_ln_fwd``: a two-pass fp32
    block reduction of depth ceil(C / 256) + 8."""
    C_ = x.shape[1] if cols is None else cols
    xs = x[:, :C_]
    depth = -(-x.shape[1] // 256) + 8
    mean = xs.mean(1)
    var = ((xs - mean[:, None]) ** 2).mean(1)
    rstd = 1.0 / torch.sqrt(var + eps)
    mean_tol = 2 * (depth * U32 * xs.abs().mean(1) + 2 * U32 * mean.abs())
    var_err = 2 * ((depth + 1) * U32 * var + mean_tol ** 2 + 4 * U32 * var + U32 * eps)
    rstd_tol = 0.5 * var_err / (var + eps) + 4 * U32
    return mean, rstd, mean_tol, rstd_tol


def colsum_ref(dz, drop_last=False):
    """Column sums of dz [rows, C]; ``drop_last`` (self-check perturbation) misses the last row."""
    return (dz[:-1] if drop_last else dz).sum(0)


# ------------------------------------------------------------- the comparison helpers themselves
def test_helpers_reject_perturbed_references():
    """Each comparison accepts a faithful result and rejects a perturbed reference (CPU tensors,
    no kernel launch): a convolution with the border tap dropped, a stride-2 input gradient whose
    zero-stuffed grid is shifted by one row, a max pool breaking ties last-max, BN variance over
    rows - 1, an LN rstd over C - 1 columns, a colsum missing its last row."""
    g = gen(0)
    # convolution forward, exact: the faithful result is the reference rounded once to bf16
    X, Wm = ints(g, 2, 8, 8, 16, r=1), ints(g, 24, 144, r=1, density=0.5)
    y = conv_ref(X, Wm, 3, 1, 1).to(BF16)
    assert not exact_violations(y, conv_ref(X, Wm, 3, 1, 1)).any()
    assert exact_violations(y, conv_ref(X, Wm, 3, 1, 1, drop_border=True)).any()
    # stride-2 input gradient: the upsample + flip form equals the scatter form, and a zero-stuffed
    # grid shifted by one row is rejected; (H + 2p - k) odd: the last input row has one tap
    H = 9
    OH, OW = out_hw(H, H, 3, 2, 1)
    dZ, Wm = ints(g, 2, OH, OW, 16, r=2), ints(g, 16, 9 * 8, r=2)
    dx = conv_dx_ref(dZ, Wm, H, H, 8, 3, 2, 1)
    assert torch.equal(conv_dx_upsample_ref(dZ, Wm, H, H, 8, 3, 2, 1), dx)
    assert not exact_violations(dx.to(BF16), dx).any()
    assert exact_violations(dx.to(BF16), conv_dx_upsample_ref(dZ, Wm, H, H, 8, 3, 2, 1, shift=1)).any()
    # max pool with many ties: first-max and last-max indices differ
    Xp = ints(g, 2, 7, 7, 4, r=1)
    yf, i_first = maxpool_ref(Xp, 3, 2, 1)
    yl, i_last = maxpool_ref(Xp, 3, 2, 1, tie="last")
    assert torch.equal(yf, yl) and not torch.equal(i_first, i_last)
    # batch norm: fp32 statistics within the bound, variance over rows - 1 rejected
    x = (torch.randn(50, 40, generator=g, dtype=F64) * 0.5 + 100).to(BF16).double()
    st = bn_stats_ref(x)
    x32 = x.float()
    m32 = x32.mean(0)
    r32 = torch.rsqrt(((x32 - m32) ** 2).mean(0) + 1e-5)
    assert not bound_violations(m32, st.mean, st.mean_tol).any()
    assert not bound_violations(r32, st.rstd, st.rstd_tol * st.rstd).any()
    bad = bn_stats_ref(x, ddof=1)
    assert bound_violations(r32, bad.rstd, st.rstd_tol * bad.rstd).any()
    # layer norm: rstd over C - 1 columns rejected
    xl = torch.randn(7, 200, generator=g, dtype=F64).to(BF16).double()
    mean, rstd, mt, rt = ln_stats_ref(xl)
    xl32 = xl.float()
    rl32 = torch.rsqrt(((xl32 - xl32.mean(1, keepdim=True)) ** 2).mean(1) + 1e-12)
    assert not bound_violations(rl32, rstd, rt * rstd).any()
    assert bound_violations(rl32, ln_stats_ref(xl, cols=199)[1], rt * rstd).any()
    # column sums: a sum missing the last row rejected
    dz = ints(g, 300, 40, r=4)
    cs = dz.sum(0).float()
    assert not exact_violations(cs, colsum_ref(dz)).any()
    assert exact_violations(cs, colsum_ref(dz, drop_last=True)).any()


# ---------------------------------------------------------------------------- convolutions
class ConvCase(NamedTuple):
    name: str
    N: int
    H: int
    W: int
    cin: int
    cout: int
    k: int
    s: int
    p: int
    bias: bool
    act: int
    fwd: str          # implicit-direct | implicit-splitk | im2col | im2col-mx8
    dx: str           # flip | upsample-flip | col2im
    dw: str           # implicit weight gradient: split (split-K, sk > 1) | accumulate (sk == 1, +=); im2col: gemm
    rx: int = 1
    rw: int = 1
    dens_w: float = 1.0
    rdy: int = 1
    dens_dy: float = 1.0

    @property
    def kc(self):
        return self.k * self.k * self.cin

    @property
    def kp(self):
        return (self.kc + 7) // 8 * 8

    @property
    def implicit(self):
        return self.fwd.startswith("implicit")


CONV_CASES = [
    # implicit GEMM: 64-channel K blocks, pixel tiles of whole image rows
    ConvCase("s1_64x64_32x32_bias_relu", 2, 32, 32, 64, 64, 3, 1, 1, True, ACT_RELU,
             "implicit-direct", "flip", "split", dens_w=0.3),
    ConvCase("s1_64x64_32x32", 2, 32, 32, 64, 64, 3, 1, 1, False, ACT_NONE,
             "implicit-splitk", "flip", "split", dens_w=0.3),
    ConvCase("s2_64x128_32x32_odd_tail", 2, 32, 32, 64, 128, 3, 2, 1, True, ACT_RELU,
             "implicit-direct", "upsample-flip", "split", dens_w=0.3),
    ConvCase("1x1_s2_downsample_16x16", 4, 16, 16, 64, 128, 1, 2, 0, False, ACT_NONE,
             "implicit-direct", "upsample-flip", "split"),
    ConvCase("5x5_p2_16x16", 2, 16, 16, 64, 64, 5, 1, 2, False, ACT_NONE,
             "implicit-splitk", "flip", "split", dens_w=0.12),
    ConvCase("nonsquare_8x16", 3, 8, 16, 64, 64, 3, 1, 1, True, ACT_NONE,
             "implicit-direct", "flip", "split", dens_w=0.3),
    ConvCase("4x4_N5_tile_past_N", 5, 4, 4, 64, 64, 3, 1, 1, True, ACT_RELU,
             "implicit-direct", "flip", "accumulate", dens_w=0.3),
    ConvCase("2x2_images", 3, 2, 2, 64, 64, 3, 1, 1, True, ACT_NONE,
             "implicit-direct", "flip", "accumulate", dens_w=0.3),
    ConvCase("cout96_col2im", 4, 8, 8, 64, 96, 3, 1, 1, True, ACT_RELU,
             "implicit-direct", "col2im", "split", dens_w=0.3),
    ConvCase("cout192_n_tail", 6, 8, 8, 64, 192, 3, 1, 1, True, ACT_RELU,
             "implicit-direct", "flip", "split", dens_w=0.25, dens_dy=0.5),
    ConvCase("512x512_4x4", 8, 4, 4, 512, 512, 3, 1, 1, False, ACT_NONE,
             "implicit-splitk", "flip", "accumulate", dens_w=0.04, dens_dy=0.5),
    # im2col + GEMM + col2im
    ConvCase("lenet_conv1_3x8_k5", 2, 32, 32, 3, 8, 5, 1, 0, True, ACT_RELU,
             "im2col", "col2im", "gemm", rx=2),
    ConvCase("lenet_conv2_8x16_14x14", 3, 14, 14, 8, 16, 5, 1, 0, True, ACT_RELU,
             "im2col", "col2im", "gemm", dens_w=0.6),
    ConvCase("resnet_stem_3x64_k3", 2, 32, 32, 3, 64, 3, 1, 1, True, ACT_NONE,
             "im2col", "col2im", "gemm", rx=4, dens_w=0.4),
    ConvCase("cin6_s2_p2_7x10", 3, 7, 10, 6, 16, 3, 2, 2, True, ACT_RELU,
             "im2col", "col2im", "gemm", rx=2, rw=2),
    ConvCase("gelu_aux_out", 2, 8, 8, 8, 24, 3, 1, 1, True, ACT_GELU,
             "im2col", "col2im", "gemm"),
    ConvCase("mx8_forward", 2, 16, 16, 3, 16, 3, 1, 1, True, ACT_RELU,
             "im2col-mx8", "col2im", "gemm", rx=4, rw=2),
]


def conv_id(c):
    return f"{c.name}-{c.fwd}-dx_{c.dx}-dw_{c.dw}"


def conv_operands(c: ConvCase, seed=0):
    """x [N, H, W, Cin], w [Cout, Kp] (pad columns zero), bias [Cout] or None, dy [N, OH, OW, Cout]:
    float64 CPU integers, the same on every machine."""
    g = gen(1000 + seed + CONV_CASES.index(c))
    OH, OW = out_hw(c.H, c.W, c.k, c.s, c.p)
    X = ints(g, c.N, c.H, c.W, c.cin, r=c.rx)
    Wm = torch.zeros(c.cout, c.kp, dtype=F64)
    Wm[:, :c.kc] = ints(g, c.cout, c.kc, r=c.rw, density=c.dens_w)
    b = ints(g, c.cout, r=4) if c.bias else None
    dY = ints(g, c.N, OH, OW, c.cout, r=c.rdy, density=c.dens_dy)
    return X, Wm, b, dY


@pytest.mark.parametrize("c", CONV_CASES, ids=conv_id)
def test_conv_operands_are_exact(c):
    """Exactness guard: from each case's integer operands, every value the kernel path stores in
    bf16 (y, the GELU pre-activation, dz, the fallback's dcol, dx) is an integer of magnitude
    <= 256, and every fp32 sum (split-K workspace, gw after two backward passes, gb) stays below
    2^24, so the bit-exact comparisons of ``test_conv`` are legitimate.  The bounds are the same
    formulas on |operands|, so they hold for every partial sum."""
    X, Wm, b, dY = conv_operands(c)
    aX, aW, adY = X.abs(), Wm.abs(), dY.abs()
    yabs = conv_ref(aX, aW, c.k, c.s, c.p) + (b.abs() if b is not None else 0)
    assert float(yabs.max()) <= BF16_INT, f"y / pre-activation: {float(yabs.max())}"
    assert float(adY.max()) <= BF16_INT                       # dz = dy * relu'(y)
    dz_max = 1.13 if c.act == ACT_GELU else 1.0               # max |gelu'| < 1.13
    if c.dx == "col2im":
        dcol = adY.reshape(-1, c.cout) @ aW * dz_max
        assert float(dcol.max()) <= BF16_INT, f"dcol: {float(dcol.max())}"
    dxabs = conv_dx_ref(adY * dz_max, aW, c.H, c.W, c.cin, c.k, c.s, c.p)
    assert float(dxabs.max()) <= BF16_INT, f"dx: {float(dxabs.max())}"
    gwabs = 2 * conv_dw_ref(aX, adY * dz_max, c.k, c.s, c.p, c.kp)
    assert float(gwabs.max()) < F32_INT and float(2 * adY.sum()) < F32_INT
    if c.fwd == "im2col-mx8":
        # e4m3 under the per-32 UE8M0 scales: the quantised operands dequantise to themselves
        from bflc_demo_b200.ops.mx8 import quantize_mx8_reference
        col = im2col_ref(X, c.k, c.s, c.p)
        colp = torch.zeros(col.shape[0], c.kp, dtype=F64)
        colp[:, :c.kc] = col
        for t in (colp, Wm):
            assert torch.equal(quantize_mx8_reference(t.float()).dequantize().double(), t)


class CallLog:
    """Records the native entry points ``ops.nn`` calls (the extension module's attributes are
    wrapped for the test), so a case asserts which path ran."""
    NAMES = ("conv_gemm", "im2col", "col2im", "upsample_zero", "cast_f32_to_bf16", "gemm", "gemm2",
             "gemm_mx8", "act_bwd_colsum")

    def __init__(self, monkeypatch):
        self.log = []
        m = C()
        for name in self.NAMES:
            monkeypatch.setattr(m, name, self._wrap(name, getattr(m, name)))

    def _wrap(self, name, orig):
        def call(*a, **kw):
            # conv_gemm(mode, flip, x, other, d, N, H, W, C, OH, OW, KH, KW, stride, pad, n_out, bias, act,
            #           aux_out, aux_in, act_bwd, colsum, split_k, accumulate)
            self.log.append((name, a[0], a[1], a[22], a[23]) if name == "conv_gemm" else (name,))
            return orig(*a, **kw)
        return call

    def take(self):
        out, self.log = self.log, []
        return out


def fwd_path(log):
    names = [e[0] for e in log]
    cg = [e for e in log if e[0] == "conv_gemm"]
    if "im2col" in names:
        assert not cg, log
        return "im2col-mx8" if "gemm_mx8" in names else "im2col"
    assert len(cg) == 1 and cg[0][1:3] == (1, 0), log
    if cg[0][3] > 1:
        assert "cast_f32_to_bf16" in names, log
        return "implicit-splitk"
    return "implicit-direct"


def bwd_paths(log):
    names = [e[0] for e in log]
    cg = [e for e in log if e[0] == "conv_gemm"]
    dws = [e for e in cg if e[1] == 2]
    flips = [e for e in cg if e[1] == 1]
    if dws:
        assert len(dws) == 1, log
        _, _, _, sk, acc = dws[0]
        assert bool(acc) == (sk == 1), f"weight gradient sk={sk} must accumulate exactly when sk == 1"
        dw = "split" if sk > 1 else "accumulate"
    else:
        assert "gemm" in names or "gemm2" in names, log
        dw = "gemm"
    if "col2im" in names:
        assert not flips and "upsample_zero" not in names, log
        dx = "col2im"
    else:
        assert len(flips) == 1 and flips[0][2] == 1, log
        dx = "upsample-flip" if "upsample_zero" in names else "flip"
    return dx, dw


@gpu
@pytest.mark.parametrize("c", CONV_CASES, ids=conv_id)
def test_conv(c, monkeypatch):
    """``ops.nn.conv2d`` forward and backward against the fp64 reference, on the path the case
    names: y (bf16) and dx exact, gw and gb exact in fp32, a second backward exactly doubling
    both.  GELU: the saved pre-activation exact, y / dz / dx / gw within bounds."""
    from bflc_demo_b200.ops import nn as F
    X, Wm, b, dY = conv_operands(c)
    prev = F.set_precision("mx8" if c.fwd == "im2col-mx8" else "bf16")
    try:
        assert F.conv_is_implicit(c.H, c.W, c.cin, c.k, c.k, c.s, c.p, c.kp) == c.implicit
        calls = CallLog(monkeypatch)
        x = X.to(BF16).cuda().requires_grad_(True)
        w = Wm.to(BF16).cuda()
        bias = b.float().cuda() if b is not None else None
        gw = torch.zeros(c.cout, c.kp, device="cuda")
        gb = torch.zeros(c.cout, device="cuda") if b is not None else None
        dy = dY.to(BF16).cuda()
        y = F.conv2d(x, w, bias, gw, gb, c.k, c.k, c.s, c.p, c.act)
        assert fwd_path(calls.take()) == c.fwd
        pre = y.grad_fn.saved_tensors[2] if c.act == ACT_GELU else None
        y.backward(dy)
        assert bwd_paths(calls.take()) == (c.dx, c.dw)
        dx1, gw1 = x.grad.clone(), gw.clone()
        gb1 = gb.clone() if gb is not None else None
        x.grad = None
        F.conv2d(x, w, bias, gw, gb, c.k, c.k, c.s, c.p, c.act).backward(dy)
        torch.cuda.synchronize()
    finally:
        F.set_precision(prev)

    Xd, Wd, dYd = X.cuda(), Wm.cuda(), dY.cuda()
    z = conv_ref(Xd, Wd, c.k, c.s, c.p) + (b.cuda() if b is not None else 0)
    if c.act == ACT_GELU:
        assert_exact(pre, z.reshape(pre.shape), "pre-activation (aux_out)")
        assert_bound(y, gelu_ref(z), 2.0 ** -20 * (1 + z.abs()), "y = gelu(pre)")
        dgelu = gelu_grad_ref(z)
        dZ = dYd * dgelu
        # dz is stored in bf16 (half an ulp) after fp32 erff / __expf (2^-17 of |dy|)
        dz_err = (2.0 ** -8 * dZ.abs() + 2.0 ** -17 * dYd.abs())
        K = c.N * z.shape[1] * z.shape[2]
        gw_slack = conv_dw_ref(Xd.abs(), dz_err, c.k, c.s, c.p, c.kp) + \
            K * U32 * conv_dw_ref(Xd.abs(), dZ.abs(), c.k, c.s, c.p, c.kp)
        assert_bound(gw1, conv_dw_ref(Xd, dZ, c.k, c.s, c.p, c.kp), gw_slack, "gw (gelu)")
        # dx: dz error, then dcol rounded to bf16 and summed over the taps
        dxabs = conv_dx_ref(dZ.abs(), Wd.abs(), c.H, c.W, c.cin, c.k, c.s, c.p)
        dx_slack = conv_dx_ref(dz_err, Wd.abs(), c.H, c.W, c.cin, c.k, c.s, c.p) + 2.0 ** -8 * dxabs \
            + c.cout * U32 * dxabs
        assert_bound(dx1, conv_dx_ref(dZ, Wd, c.H, c.W, c.cin, c.k, c.s, c.p), dx_slack, "dx (gelu)")
        assert_bound(gb1, dZ.sum((0, 1, 2)), dz_err.sum((0, 1, 2)) / 2 + K * U32 * dZ.abs().sum((0, 1, 2)),
                     "gb (gelu)")
        return
    y_ref = torch.relu(z) if c.act == ACT_RELU else z
    assert_exact(y, y_ref, "y")
    dZ = dYd * (y_ref > 0) if c.act == ACT_RELU else dYd
    dx_ref = conv_dx_ref(dZ, Wd, c.H, c.W, c.cin, c.k, c.s, c.p)
    assert_exact(dx1, dx_ref, "dx")
    if c.name.startswith("1x1_s2"):
        assert bool((dx1[:, 1::2] == 0).all()) and bool((dx1[:, :, 1::2] == 0).all()), \
            "rows / columns no output reads must get 0"
    gw_ref = conv_dw_ref(Xd, dZ, c.k, c.s, c.p, c.kp)
    assert_exact(gw1, gw_ref, "gw")
    assert_exact(gw, 2 * gw_ref, "gw after a second backward")
    if b is not None:
        assert_exact(gb1, dZ.sum((0, 1, 2)), "gb")
        assert_exact(gb, 2 * dZ.sum((0, 1, 2)), "gb after a second backward")


# ------------------------------------------------------------- im2col / col2im / upsample / transpose
IM2COL_CASES = [  # N, H, W, C, k, s, p, extra ld columns
    (2, 9, 7, 3, 3, 1, 1, 5), (1, 8, 8, 8, 5, 1, 0, 8), (3, 7, 10, 6, 3, 2, 2, 0), (2, 11, 6, 4, 4, 3, 1, 3),
    (1, 1, 1, 5, 3, 1, 1, 1),
]


@gpu
@pytest.mark.parametrize("N,H,W,Cc,k,s,p,extra", IM2COL_CASES)
def test_im2col_col2im(N, H, W, Cc, k, s, p, extra):
    """im2col bit-exact with ``ld_col > k*k*C`` (the pad columns keep their sentinel); col2im sums
    integer columns exactly and ignores the pad columns (they hold a large sentinel)."""
    g = gen(2000 + H * W + k)
    OH, OW = out_hw(H, W, k, s, p)
    kc = k * k * Cc
    X = torch.randn(N, H, W, Cc, generator=g).to(BF16)
    col = torch.full((N * OH * OW, kc + extra), 7.0, device="cuda", dtype=BF16)
    C().im2col(X.cuda(), col, N, Cc, H, W, k, k, s, p, OH, OW)
    assert torch.equal(col[:, :kc].cpu(), im2col_ref(X.double(), k, s, p).to(BF16)), "im2col"
    assert bool((col[:, kc:] == 7.0).all()), "im2col wrote pad columns"
    colv = ints(g, N * OH * OW, kc + extra, r=4)
    colv[:, kc:] = 1000.0
    dx = torch.full((N, H, W, Cc), 7.0, device="cuda", dtype=BF16)
    C().col2im(colv.to(BF16).cuda(), dx, N, Cc, H, W, k, k, s, p, OH, OW)
    assert_exact(dx, col2im_ref(colv, N, H, W, Cc, k, s, p), "col2im")


@gpu
@pytest.mark.parametrize("N,H,W,Cc,k,s,p", [(2, 32, 32, 64, 3, 2, 1), (3, 16, 16, 128, 1, 2, 0),
                                             (2, 9, 10, 8, 3, 2, 1), (1, 10, 7, 16, 3, 3, 1)])
def test_upsample_zero(N, H, W, Cc, k, s, p):
    g = gen(2100 + H + W + s)
    OH, OW = out_hw(H, W, k, s, p)
    dy = torch.randn(N, OH, OW, Cc, generator=g).to(BF16)
    up = torch.full((N, H, W, Cc), 7.0, device="cuda", dtype=BF16)
    C().upsample_zero(dy.cuda(), up, N, H, W, OH, OW, Cc, s)
    ref = torch.zeros(N, H, W, Cc, dtype=BF16)
    ref[:, 0:s * OH:s, 0:s * OW:s] = dy[:, :(H - 1) // s + 1, :(W - 1) // s + 1]
    assert torch.equal(up.cpu(), ref)


@gpu
def test_upsample_zero_rejects_channels_not_multiple_of_8():
    dy = torch.ones(1, 4, 4, 12, device="cuda", dtype=BF16)
    up = torch.full((1, 8, 8, 12), 7.0, device="cuda", dtype=BF16)
    n0 = launches()
    with pytest.raises(RuntimeError, match="invalid argument"):
        C().upsample_zero(dy, up, 1, 8, 8, 4, 4, 12, 2)
    assert launches() == n0 and bool((up == 7.0).all())


@gpu
@pytest.mark.parametrize("d3", [1, 3, 64])
@pytest.mark.parametrize("d0,d1,d2", [(1, 5, 7), (3, 13, 4), (2, 128, 12)])
def test_transpose_0213(d0, d1, d2, d3):
    g = gen(2200 + d0 + d1 + d2 + d3)
    x = torch.randn(d0, d1, d2, d3, generator=g).to(BF16).cuda()
    y = torch.full((d0, d2, d1, d3), 7.0, device="cuda", dtype=BF16)
    C().transpose_0213(x, y, d0, d1, d2, d3)
    assert torch.equal(y, x.permute(0, 2, 1, 3))
    back = torch.empty_like(x)
    C().transpose_0213(y, back, d0, d2, d1, d3)
    assert torch.equal(back, x)


# ----------------------------------------------------------------------------------- pooling
@gpu
@pytest.mark.parametrize("N,H,W,Cc,k,s,p", [(2, 7, 7, 16, 2, 2, 0), (3, 9, 8, 40, 2, 2, 0),
                                             (2, 8, 8, 16, 3, 2, 1), (2, 15, 11, 24, 3, 2, 1)],
                         ids=["k2s2_odd7", "k2s2_9x8", "k3s2p1_8x8", "k3s2p1_15x11"])
def test_maxpool(N, H, W, Cc, k, s, p):
    """Ties everywhere (integers in [-1, 1]) and -inf inputs, including a window that is -inf
    throughout: y and idx exact (first max in scan order), dx exact through the fp32 atomics of
    overlapping windows."""
    from bflc_demo_b200.ops import nn as F
    g = gen(2300 + H * W + k)
    X = ints(g, N, H, W, Cc, r=1)
    X[0, :, :, 0] = -math.inf                        # one channel of -inf
    X[1, 0:k, 0:k, 1] = -math.inf                    # a window of -inf only
    X[:, ::3, ::2, 2] = -math.inf
    y_ref, i_ref = maxpool_ref(X, k, s, p)
    x = X.to(BF16).cuda().requires_grad_(True)
    y = F.maxpool2d(x, k, s, p)
    idx = y.grad_fn.saved_tensors[0]
    assert torch.equal(idx.cpu().long(), i_ref), "argmax index (first maximum in scan order)"
    assert torch.equal(y.float().cpu().double(), y_ref)
    dY = ints(g, *y.shape, r=8)
    y.backward(dY.to(BF16).cuda())
    assert_exact(x.grad, maxpool_dx_ref(dY, i_ref, H, W, Cc), "dx")


@gpu
@pytest.mark.parametrize("H,W", [(1, 1), (2, 2), (4, 4), (7, 7)])
def test_global_avgpool(H, W):
    """Exact for HW = 1, 4, 16 on integers (a power-of-two divisor); HW = 49 within the fp32
    error of the quotient.  Backward: dy / HW."""
    from bflc_demo_b200.ops import nn as F
    g = gen(2400 + H)
    N, Cc, HW = 3, 40, H * W
    X = ints(g, N, H, W, Cc, r=8)
    x = X.to(BF16).cuda().requires_grad_(True)
    y = F.global_avgpool(x)
    dY = ints(g, N, Cc, r=100)
    y.backward(dY.to(BF16).cuda())
    ref, dref = X.mean((1, 2)), (dY / HW)[:, None, None, :].expand(N, H, W, Cc)
    if HW & (HW - 1) == 0:
        assert_exact(y, ref, "avgpool y")
        assert_exact(x.grad, dref, "avgpool dx")
    else:
        # one division, which --use_fast_math computes within 2 ulp
        assert_bound(y, ref, 8 * U32 * ref.abs(), "avgpool y")
        assert_bound(x.grad, dref, 8 * U32 * dref.abs(), "avgpool dx")


# -------------------------------------------------------------------------------- batch norm
BN_KINDS = [(0.0, 1.0), (100.0, 0.5), (3.0, 0.02), (-256.0, 1.0), (4.0, 0.1), (5.0, 0.0)]  # (mean, std)


def bn_input(rows, Cc, seed):
    """Channels of three kinds: centred, offset (mean / std up to 256) and constant (std 0)."""
    g = gen(seed)
    mean = torch.tensor([BN_KINDS[c % len(BN_KINDS)][0] for c in range(Cc)], dtype=F64)
    std = torch.tensor([BN_KINDS[c % len(BN_KINDS)][1] for c in range(Cc)], dtype=F64)
    return (mean + std * torch.randn(rows, Cc, generator=g, dtype=F64)).to(BF16).double()


@gpu
@pytest.mark.parametrize("relu,res", [(False, False), (True, False), (False, True), (True, True)],
                         ids=["plain", "relu", "res", "relu_res"])
@pytest.mark.parametrize("Cc", [32, 40, 200, 512])
@pytest.mark.parametrize("rows", [1, 50, 384, 16384])
def test_batchnorm_train(rows, Cc, relu, res):
    """Training-mode ``ops.nn.batchnorm``: fp32 mean / rstd against fp64 (rstd within 2^-14
    relative or the tighter accumulation bound), running statistics (momentum 0.1, unbiased
    variance; rows = 1 skips the correction), y, dx, dres in bf16 and dgamma / dbeta in fp32 (zero
    on entry, as the kernel requires)."""
    from bflc_demo_b200.ops import nn as F
    X = bn_input(rows, Cc, 3000 + rows + Cc)
    g = gen(3100 + rows + Cc)
    gamma = (0.5 + torch.rand(Cc, generator=g, dtype=F64)).float().double()
    beta = torch.randn(Cc, generator=g, dtype=F64).float().double()
    R = ints(g, rows, Cc, r=2) if res else None
    dY = ints(g, rows, Cc, r=4)
    rm0 = torch.randn(Cc, generator=g, dtype=F64).float().double()
    rv0 = (0.5 + torch.rand(Cc, generator=g, dtype=F64)).float().double()
    dev = "cuda"
    x = X.to(BF16).to(dev).requires_grad_(True)
    r = R.to(BF16).to(dev).requires_grad_(True) if res else None
    rm, rv = rm0.float().to(dev), rv0.float().to(dev)
    gg, gbt = torch.zeros(Cc, device=dev), torch.zeros(Cc, device=dev)
    y = F.batchnorm(x, gamma.float().to(dev), beta.float().to(dev), gg, gbt, rm, rv, True, relu, r)
    _, _, _, mean_k, rstd_k = y.grad_fn.saved_tensors
    y.backward(dY.to(BF16).to(dev))
    torch.cuda.synchronize()

    Xd = X.to(dev)
    st = bn_stats_ref(Xd)
    assert_bound(mean_k, st.mean, st.mean_tol, "mean")
    assert_bound(rstd_k, st.rstd, st.rstd_tol * st.rstd, "rstd")
    var_tol = 2 * st.rstd_tol * (st.var + 1e-5)
    unb = st.var * rows / (rows - 1) if rows > 1 else st.var
    unb_tol = var_tol * (rows / (rows - 1) if rows > 1 else 1)
    rm_ref = 0.9 * rm0.to(dev) + 0.1 * st.mean
    rv_ref = 0.9 * rv0.to(dev) + 0.1 * unb
    assert_bound(rm, rm_ref, 0.1 * st.mean_tol + 4 * U32 * (rm0.to(dev).abs() + 0.1 * st.mean.abs()), "run_mean")
    assert_bound(rv, rv_ref, 0.1 * unb_tol + 4 * U32 * (rv0.to(dev).abs() + 0.1 * unb), "run_var")

    gam, bet = gamma.to(dev), beta.to(dev)
    xc = Xd - st.mean
    xhat = xc * st.rstd
    pre = xhat * gam + bet + (R.to(dev) if res else 0)
    y_ref = torch.relu(pre) if relu else pre
    xhat_err = xc.abs() * st.rstd * st.rstd_tol + st.rstd * st.mean_tol + 2 * U32 * xhat.abs()
    y_slack = gam * xhat_err + 4 * U32 * (xhat.abs() * gam + bet.abs() + (R.to(dev).abs() if res else 0))
    assert_bound(y, y_ref, y_slack, "y")

    # backward: the ReLU mask is the kernel's own y > 0
    gmask = (y.detach().double() > 0) if relu else torch.ones_like(Xd, dtype=torch.bool)
    G_ = dY.to(dev) * gmask
    depth = rows_per_lane(rows, grid_y(rows, 64))
    dbeta_ref = G_.sum(0)
    dgamma_ref = (G_ * xhat).sum(0)
    assert_exact(gbt, dbeta_ref, "dbeta")
    dgamma_tol = depth * U32 * (G_ * xhat).abs().sum(0) + (G_.abs() * xhat_err).sum(0)
    assert_bound(gg, dgamma_ref, dgamma_tol, "dgamma")
    if res:
        assert_exact(r.grad, G_, "dres")
    dx_ref = gam * st.rstd * (G_ - (dbeta_ref + xhat * dgamma_ref) / rows)
    dx_slack = gam * st.rstd * ((xhat.abs() * dgamma_tol + dgamma_ref.abs() * xhat_err) / rows
                                + 8 * U32 * (G_.abs() + (dbeta_ref.abs() + (xhat * dgamma_ref).abs()) / rows)) \
        + dx_ref.abs() * st.rstd_tol
    assert_bound(x.grad, dx_ref, dx_slack, "dx")


@gpu
@pytest.mark.parametrize("relu,res", [(False, False), (True, True)], ids=["plain", "relu_res"])
def test_batchnorm_eval(relu, res):
    """Eval mode normalises with the running statistics (rstd = rsqrt(run_var + 1e-5) in fp32)
    and leaves them unchanged."""
    from bflc_demo_b200.ops import nn as F
    rows, Cc = 384, 200
    X = bn_input(rows, Cc, 3200)
    g = gen(3201)
    gamma = (0.5 + torch.rand(Cc, generator=g, dtype=F64)).float().cuda()
    beta = torch.randn(Cc, generator=g, dtype=F64).float().cuda()
    R = ints(g, rows, Cc, r=2).cuda() if res else None
    rm = torch.tensor([BN_KINDS[c % len(BN_KINDS)][0] for c in range(Cc)], dtype=F32).cuda() + 0.25
    rv = (0.5 + torch.rand(Cc, generator=g)).cuda()
    rm0, rv0 = rm.clone(), rv.clone()
    y = F.batchnorm(X.to(BF16).cuda(), gamma, beta, None, None, rm, rv, False, relu,
                    R.to(BF16) if res else None)
    assert torch.equal(rm, rm0) and torch.equal(rv, rv0)
    rstd = torch.rsqrt(rv + 1e-5).double()
    xhat = (X.cuda() - rm.double()) * rstd
    pre = xhat * gamma.double() + beta.double() + (R if res else 0)
    ref = torch.relu(pre) if relu else pre
    slack = 4 * U32 * (xhat.abs() * gamma.double() + beta.double().abs() + (R.abs() if res else 0))
    assert_bound(y, ref, slack, "eval y")


# -------------------------------------------------------------------------------- layer norm
@gpu
@pytest.mark.parametrize("Cc", [64, 200, 256, 768, 1000, 1024])
@pytest.mark.parametrize("rows", [1, 7, 300, 2000])
def test_layernorm(rows, Cc):
    """``ops.nn.layernorm``: fp32 mean / rstd, bf16 y and dx against fp64, dgamma / dbeta added
    (``+=``) into nonzero values; the last row is constant, which gives y = beta (eps 1e-12).
    2000 rows run the forward's (1056) and backward's (264) grid-stride loops."""
    from bflc_demo_b200.ops import nn as F
    g = gen(4000 + rows + Cc)
    X = (torch.randn(rows, Cc, generator=g, dtype=F64) * 2 + torch.randn(rows, 1, generator=g, dtype=F64) * 4)
    X[-1] = 1.5
    X = X.to(BF16).double()
    gamma = (0.5 + torch.rand(Cc, generator=g, dtype=F64)).float().double()
    beta = torch.randn(Cc, generator=g, dtype=F64).float().double()
    dY = ints(g, rows, Cc, r=4)
    gg0, gb0 = ints(g, Cc, r=100), ints(g, Cc, r=100)
    x = X.to(BF16).cuda().requires_grad_(True)
    gg, gb = gg0.float().cuda(), gb0.float().cuda()
    y = F.layernorm(x, gamma.float().cuda(), beta.float().cuda(), gg, gb)
    _, _, mean_k, rstd_k = y.grad_fn.saved_tensors
    y.backward(dY.to(BF16).cuda())
    torch.cuda.synchronize()

    Xd, gam, bet, dYd = X.cuda(), gamma.cuda(), beta.cuda(), dY.cuda()
    mean, rstd, mt, rt = ln_stats_ref(Xd)
    assert_bound(mean_k, mean, mt, "mean")
    assert_bound(rstd_k, rstd, rt * rstd, "rstd")
    assert torch.equal(y[-1].float().double(), bet.to(BF16).double()), "constant row: y = beta"
    xc = Xd - mean[:, None]
    xhat = xc * rstd[:, None]
    xhat_err = (xc.abs() * rt[:, None] + mt[:, None]) * rstd[:, None] + 2 * U32 * xhat.abs()
    assert_bound(y, xhat * gam + bet, gam * xhat_err + 4 * U32 * (xhat.abs() * gam + bet.abs()), "y")
    # backward on the rows with a nonzero variance; the constant row's rstd is 1e6
    gy = dYd * gam
    s1, s2 = gy.mean(1, keepdim=True), (gy * xhat).mean(1, keepdim=True)
    dx_ref = rstd[:, None] * (gy - s1 - xhat * s2)
    depth = -(-Cc // 256) + 8
    s2_tol = (depth * U32 * (gy * xhat).abs().sum(1, keepdim=True) + (gy.abs() * xhat_err).sum(1, keepdim=True)) / Cc
    s1_tol = depth * U32 * gy.abs().sum(1, keepdim=True) / Cc
    dx_slack = rstd[:, None] * (s1_tol + xhat.abs() * s2_tol + xhat_err * s2.abs()
                                + 6 * U32 * (gy.abs() + s1.abs() + (xhat * s2).abs())) + dx_ref.abs() * rt[:, None]
    assert_bound(x.grad[:-1], dx_ref[:-1], dx_slack[:-1], "dx")
    grid = min(rows, 264)
    gdepth = -(-rows // grid) + grid + 1
    assert_exact(gb, gb0.cuda() + dYd.sum(0), "dbeta += sum dy")
    # the constant row's xhat is exactly 0 (its mean is exact, checked by y = beta above)
    dg_ref = gg0.cuda() + (dYd * xhat)[:-1].sum(0)
    dg_tol = gdepth * U32 * (gg0.cuda().abs() + (dYd * xhat)[:-1].abs().sum(0)) + (dYd.abs() * xhat_err)[:-1].sum(0)
    assert_bound(gg, dg_ref, dg_tol, "dgamma += sum dy * xhat")


@gpu
def test_layernorm_bwd_rejects_more_than_1024_columns():
    rows, Cc = 4, 1025
    t = torch.zeros(rows, Cc, device="cuda", dtype=BF16)
    f = torch.zeros(Cc, device="cuda")
    st = torch.zeros(rows, device="cuda")
    dx = torch.full((rows, Cc), 7.0, device="cuda", dtype=BF16)
    n0 = launches()
    with pytest.raises(RuntimeError, match="invalid argument"):
        C().layernorm_bwd(t, t, f, st, st, dx, f.clone(), f.clone(), rows, Cc)
    assert launches() == n0 and bool((dx == 7.0).all())


# ------------------------------------------------------------------------------- row softmax
@gpu
@pytest.mark.parametrize("scale", [1.0, 0.125])
@pytest.mark.parametrize("cols", [1, 17, 32, 33, 128, 200, 512])
def test_softmax_rows(cols, scale):
    """Row softmax fwd / bwd on 37 rows: random, large-magnitude and partially -inf rows.  Bound:
    ``__expf`` and the fp32 sum (relative to p) plus half a bf16 ulp.  An all -inf row gives NaN
    (no caller produces one); it is recorded here, not relied on."""
    g = gen(5000 + cols)
    rows = 37
    X = torch.randn(rows, cols, generator=g, dtype=F64) * 3
    X[1] *= 300                                            # large magnitude: |x| ~ 1000
    X[2, ::3] = -math.inf                                  # partially -inf (cols == 1: the NaN row)
    X[3, 1:] = -math.inf                                   # one finite entry: p = 1
    X[4] = -math.inf
    xb = X.to(BF16)
    y = torch.full((rows, cols), 7.0, device="cuda", dtype=BF16)
    C().softmax_fwd(xb.cuda(), y, rows, cols, scale)
    assert bool(torch.isnan(y[4].float()).all()), "all -inf row"
    ok = torch.ones(rows, dtype=torch.bool)
    ok[4] = False
    if cols == 1:
        ok[2] = False                                       # the row is all -inf too
    t = xb.double() * scale
    ref = torch.softmax(t[ok], 1)
    mx = t[ok].max(1, keepdim=True).values
    arg = (t[ok] - mx).abs().nan_to_num(posinf=0)
    assert_bound(y[ok.cuda()], ref, ref * (2.0 ** -20 + 4 * U32 * arg + 2 * cols * U32), "softmax fwd")
    # backward on the kernel's own probabilities
    P = y[ok.cuda()].double()
    dY = torch.randn(int(ok.sum()), cols, generator=g, dtype=F64).to(BF16).double()
    dx = torch.empty(int(ok.sum()), cols, device="cuda", dtype=BF16)
    C().softmax_bwd(dY.to(BF16).cuda(), P.to(BF16), dx, P.shape[0], cols, scale)
    dYd = dY.cuda()
    dot = (dYd * P).sum(1, keepdim=True)
    ref = scale * P * (dYd - dot)
    slack = scale * P * (cols * U32 * (dYd * P).abs().sum(1, keepdim=True) + 3 * U32 * (dYd.abs() + dot.abs()))
    assert_bound(dx, ref, slack, "softmax bwd")


# -------------------------------------------------------------------------------- embeddings
@gpu
@pytest.mark.parametrize("mode", ["seq", "pos_ids", "no_pos", "one_id"])
def test_embedding(mode):
    """Forward bit-equal to (table[ids] + pos[p]) rounded once; backward with integer dy exact in
    fp32: positions r % seq, packed rows with ``pos_ids``, no position table, every row on one
    id (contention on one table row's atomics)."""
    from bflc_demo_b200.ops import nn as F
    g = gen(6000 + len(mode))
    V, Cc, seq, rows = 50, 72, 16, 16 * 9
    ids = torch.randint(0, V, (rows,), generator=g, dtype=torch.int32)
    if mode == "one_id":
        ids[:] = 7
    table = torch.randn(V, Cc, generator=g).to(BF16)
    pos = torch.randn(seq, Cc, generator=g).to(BF16) if mode != "no_pos" else None
    pos_ids = torch.randint(0, seq, (rows,), generator=g, dtype=torch.int32) if mode == "pos_ids" else None
    p = pos_ids.long() if pos_ids is not None else torch.arange(rows) % seq
    gt0 = ints(g, V, Cc, r=50)
    gt = gt0.float().cuda()
    gp = torch.zeros(seq, Cc, device="cuda") if pos is not None else None
    out = F.embedding(ids.cuda(), table.cuda(), pos.cuda() if pos is not None else None, gt, gp, seq,
                      pos_ids.cuda() if pos_ids is not None else None)
    ref = table[ids.long()].float() + (pos[p].float() if pos is not None else 0)
    assert torch.equal(out.cpu(), ref.to(BF16))
    dY = ints(g, rows, Cc, r=8)
    out.backward(dY.to(BF16).cuda())
    assert_exact(gt, gt0.index_add(0, ids.long(), dY), "dtable")
    if pos is not None:
        assert_exact(gp, torch.zeros(seq, Cc, dtype=F64).index_add(0, p, dY), "dpos")


# -------------------------------------------------------------------------------- act_bwd_colsum
@gpu
@pytest.mark.parametrize("outputs", ["dz_colsum", "dz", "colsum"])
@pytest.mark.parametrize("mode", [0, 1, 2], ids=["identity", "relu", "gelu"])
@pytest.mark.parametrize("rows,Cc", [(37, 8), (300, 40), (9000, 40), (8500, 768)])
def test_act_bwd_colsum(rows, Cc, mode, outputs):
    """dz = dy * act'(aux) and colsum += sum over rows (into nonzero values); rows above 8192
    reach the grid-y cap of 128.  ReLU's mask is aux > 0, so +0 and -0 give 0.  GELU' against the
    fp64 erf formula; integer dy makes modes 0 and 1 exact."""
    g = gen(7000 + rows + Cc + mode)
    dY = ints(g, rows, Cc, r=8)
    aux = torch.randn(rows, Cc, generator=g).to(BF16)
    aux[::5, ::3] = 0.0
    aux[1::5, ::3] = -0.0
    c0 = ints(g, Cc, r=1000)
    dz = torch.full((rows, Cc), 7.0, device="cuda", dtype=BF16) if "dz" in outputs else None
    cs = c0.float().cuda() if "colsum" in outputs else None
    C().act_bwd_colsum(dY.to(BF16).cuda(), aux.cuda() if mode else None, dz, cs, rows, Cc, mode)
    a = aux.double().cuda()
    dYd = dY.cuda()
    if mode == 0:
        ref = dYd
    elif mode == 1:
        ref = dYd * (a > 0)
    else:
        ref = dYd * gelu_grad_ref(a)
    depth = rows_per_lane(rows, grid_y(rows, 128))
    if mode < 2:
        if dz is not None:
            assert_exact(dz, ref, "dz")
        if cs is not None:
            assert_exact(cs, c0.cuda() + colsum_ref(ref), "colsum")
    else:
        err = 2.0 ** -17 * dYd.abs()                          # erff, __expf in fp32
        if dz is not None:
            assert_bound(dz, ref, err, "dz (gelu)")
        if cs is not None:
            assert_bound(cs, c0.cuda() + colsum_ref(ref),
                         err.sum(0) + depth * U32 * (c0.cuda().abs() + ref.abs().sum(0)), "colsum (gelu)")
