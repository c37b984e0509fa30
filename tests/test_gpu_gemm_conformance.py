"""Conformance of the wgmma GEMMs (``csrc/kernels/gemm_sm100.cu``, ``gemm2_sm100.cu``): every tile
width, operand layout, tail, epilogue and launch form against a float64 reference.

Two kinds of reference:

* exact -- operands are small integers (|v| <= 8, times a power of two), exact in bf16 and in
  e4m3, and K <= 2048, so every partial sum is exact in fp32.  An fp32 result must then equal the
  fp64 product bit for bit, and a bf16 / e4m3 result must equal it rounded once to nearest even.
  A dropped, doubled or misplaced K-block, row, column or tile cannot pass.
* rounding-realistic -- random-normal operands, compared elementwise with a bound of
  ``c * K * 2^-24 * (|A| @ |B|^T)`` for the fp32 accumulation plus half an ulp of the output type.

``C().gemm`` is called with an explicit ``force_bn`` (its last argument), so which
``gemm_kernel<BN, EPI>`` runs does not depend on the device's SM count; test ids name the tile
width and the operand layout (t<A MN-major><B MN-major>).  Needs an H100 (``pytest -m gpu``).
"""
import struct

import pytest
import torch

from bflc_demo_b200._native import C

pytestmark = pytest.mark.gpu

BF16, F32, E4M3 = torch.bfloat16, torch.float32, torch.float8_e4m3fn
DT = {F32: 0, BF16: 1, E4M3: 2}
EPI_GENERIC, EPI_XENT, EPI_ARGMAX = 0, 1, 2
ACT_NONE, ACT_RELU, ACT_GELU = 0, 1, 2
U32 = 2.0 ** -24                                          # fp32 unit roundoff
HALF_ULP = {F32: 2.0 ** -24, BF16: 2.0 ** -8, E4M3: 2.0 ** -4}   # relative, normal range
FLOOR = {F32: 2.0 ** -126, BF16: 2.0 ** -126, E4M3: 2.0 ** -10}  # absolute: subnormal spacing
LAYOUTS = {"t00": (False, False), "t01": (False, True), "t10": (True, False), "t11": (True, True)}


# ------------------------------------------------------------------------------------ helpers
def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def ints(g, *shape, r=8, dev="cuda"):
    """float64 tensor of integers in [-r, r]."""
    return torch.randint(-r, r + 1, shape, generator=g, device=dev).double()


def padded(t, dtype, extra=0, fill=3.0):
    """``t`` stored as ``dtype`` in rows padded to a 16-byte multiple (+ ``extra`` elements) and
    sliced back to its width, as padded-and-sliced activations are: the row stride is not the
    width.  The pad holds ``fill``, so a kernel reading past the width changes its result."""
    es = 1 if dtype == E4M3 else 2
    c = t.shape[-1]
    cp = (c + 16 // es - 1) // (16 // es) * (16 // es) + extra
    if dtype == E4M3:
        s = torch.full((*t.shape[:-1], cp), fill, device=t.device).to(E4M3).view(torch.uint8)
        s[..., :c] = t.float().to(E4M3).view(torch.uint8)
        return s.view(E4M3)[..., :c]
    s = torch.full((*t.shape[:-1], cp), fill, device=t.device, dtype=dtype)
    s[..., :c] = t.to(dtype)
    return s[..., :c]


def operands(A, B, a_mn, b_mn, dtype=BF16, extra=0):
    """Logical A [.., M, K] and B [.., N, K] stored K-major, or MN-major as [.., K, M|N]."""
    a = padded(A.transpose(-1, -2) if a_mn else A, dtype, extra)
    b = padded(B.transpose(-1, -2) if b_mn else B, dtype, extra)
    return a, b


def gemm(a, b, d, M, N, K, *, bn, batch=1, a_mn=False, b_mn=False, a_bs=0, b_bs=0, epi=EPI_GENERIC,
         d_dtype=None, ldd=None, d_bs=0, alpha=1.0, bias=None, act=ACT_NONE, aux_out=None,
         aux_in=None, act_bwd=0, colsum=None, split_k=1, accumulate=False, labels=None, labels_bs=0,
         grad_scale=1.0, loss_sum=None, correct=None, b_maps=None, bias_ptrs=None, dyn_ptr=0):
    """One ``gemm_sm100`` launch through the binding, with the N-tile pinned to ``bn``."""
    if d_dtype is None:
        d_dtype = DT[d.dtype] if d is not None else 1
    if ldd is None:
        ldd = d.stride(-2) if d is not None else 0
    C().gemm(a, b, d, M, N, K, batch, a.stride(-2), b.stride(-2), a_bs, b_bs, a_mn, b_mn,
             a.dtype == E4M3, epi, d_dtype, ldd, d_bs, alpha, bias, act, aux_out, aux_in, act_bwd,
             colsum, split_k, accumulate, labels, labels_bs, grad_scale, loss_sum, correct, b_maps,
             bias_ptrs, 0, 0, 0, 0, dyn_ptr, bn)


def exact_violations(out, ref):
    """Elements of ``out`` that differ from ``ref`` (float64, exact in fp32) rounded once to
    ``out``'s type.  Raises if the reference itself is not exact in fp32."""
    r32 = ref.to(F32)
    assert torch.equal(r32.double(), ref), "exact reference needs fp32-exact values"
    want = r32.to(out.dtype).float() if out.dtype != F32 else r32
    return out.float() != want


def bound_violations(out, ref, acc_bound):
    """Elements with ``|out - ref| > acc_bound + half an ulp of out's type at |ref|``."""
    tol = acc_bound + HALF_ULP[out.dtype] * ref.abs() * (1 + 2.0 ** -10) + FLOOR[out.dtype]
    o = out.double()
    return ~torch.isfinite(o) | ((o - ref).abs() > tol)


def acc_bound(A, B, K, alpha=1.0, c=2.0):
    """fp32 accumulation bound c * K * 2^-24 * |alpha| * (|A| @ |B|^T), elementwise."""
    return c * K * U32 * abs(alpha) * (A.abs() @ B.abs().transpose(-1, -2))


def _report(bad, what):
    n = int(bad.sum())
    if n:
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: {n} of {bad.numel()} elements wrong, first at {idx}")


def assert_exact(out, ref, what):
    _report(exact_violations(out, ref), what)


def assert_bound(out, ref, bound, what):
    _report(bound_violations(out, ref, bound), what)


def launches():
    return C().launch_count()


# ------------------------------------------------------------- the comparison helpers themselves
def test_helpers_reject_perturbed_references():
    """The two comparisons accept a faithful result and reject references with the last K-block
    dropped, one 128 x 64 operand tile read transposed, or one output row zeroed (CPU tensors,
    no kernel launch)."""
    g = torch.Generator().manual_seed(0)
    M, N, K = 256, 192, 320
    for kind in ("exact", "bound"):
        if kind == "exact":
            A = torch.randint(-8, 9, (M, K), generator=g).double()
            B = torch.randint(-8, 9, (N, K), generator=g).double()
        else:
            A = torch.randn(M, K, generator=g, dtype=torch.float64)
            B = torch.randn(N, K, generator=g, dtype=torch.float64)
        out = (A @ B.t()).to(F32)       # a faithful kernel: fp32 result of the same product
        bound = acc_bound(A, B, K)

        def rejects(ref):
            bad = exact_violations(out, ref) if kind == "exact" else bound_violations(out, ref, bound)
            return bool(bad.any())

        assert not rejects(A @ B.t())
        assert rejects(A[:, :K - 64] @ B[:, :K - 64].t()), kind
        At = A.clone()
        At[128:256, 64:128] = A[128:256, 64:128].t().contiguous().view(128, 64)
        assert rejects(At @ B.t()), kind
        z = A @ B.t()
        z[77] = 0
        assert rejects(z), kind
        for dt in (BF16, E4M3):         # the rounded output types take the same verdicts
            o = (A @ B.t() / 64).to(F32).to(dt)
            r = A @ B.t() / 64
            if kind == "exact":
                assert not exact_violations(o, r).any()
            assert not bound_violations(o, r, bound / 64).any()
            r[5] = 0
            assert bound_violations(o, r, bound / 64).any()


# ----------------------------------------------------------------------- shape / layout sweep
SWEEP_M = [1, 127, 128, 129, 300]
SWEEP_N = {64: [8, 56, 64, 65, 130, 200], 128: [65, 128, 129, 200]}
SWEEP_K = [8, 56, 64, 72, 1000]     # 1000 = 16 K-blocks: wraps the 6-stage / 4-stage ring


@pytest.mark.parametrize("M", SWEEP_M)
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("bn", [64, 128])
def test_sweep_exact(bn, layout, M):
    """Every (N, K) of the sweep at this tile width, layout and M: fp32 and bf16 outputs exact,
    row strides from padded storage (16-byte and 32-byte pads), odd output strides, and the
    columns between N and the output stride untouched."""
    a_mn, b_mn = LAYOUTS[layout]
    g = gen(1000 * bn + 10 * M + list(LAYOUTS).index(layout))
    for i, N in enumerate(SWEEP_N[bn]):
        for j, K in enumerate(SWEEP_K):
            A, B = ints(g, M, K), ints(g, N, K)
            a, b = operands(A, B, a_mn, b_mn, extra=8 * ((i + j) % 2))
            out_dt = F32 if (i + j) % 2 == 0 else BF16
            ldd = N + (i + 2 * j) % 3
            dst = torch.full((M, ldd), 7.0, device="cuda", dtype=out_dt)
            gemm(a, b, dst, M, N, K, bn=bn, a_mn=a_mn, b_mn=b_mn, ldd=ldd)
            what = f"bn={bn} {layout} M={M} N={N} K={K} ldd={ldd} {out_dt}"
            assert_exact(dst[:, :N], A @ B.t(), what)
            assert bool((dst[:, N:] == 7.0).all()), what + ": pad columns written"


# --------------------------------------------------------------------------- generic epilogue
EM, EN, EK = 300, 200, 200          # two (BN 128) or four (BN 64) N-tiles, tails in M and K


@pytest.mark.parametrize("out_dt", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("layout", ["t00", "t11"])
@pytest.mark.parametrize("bn", [64, 128])
def test_bias_relu_alpha_colsum_exact(bn, layout, out_dt):
    a_mn, b_mn = LAYOUTS[layout]
    g = gen(11 + bn)
    A, B = ints(g, EM, EK), ints(g, EN, EK)
    bias = ints(g, EN, r=400)
    a, b = operands(A, B, a_mn, b_mn)
    d = torch.empty(EM, EN, device="cuda", dtype=out_dt)
    colsum = ints(g, EN, r=50).float()
    c0 = colsum.double().clone()
    gemm(a, b, d, EM, EN, EK, bn=bn, a_mn=a_mn, b_mn=b_mn, alpha=0.5, bias=bias.float(),
         act=ACT_RELU, colsum=colsum)
    ref = torch.relu(0.5 * (A @ B.t()) + bias)
    assert_exact(d, ref, "relu(0.5 A B^T + bias)")
    assert_exact(colsum, c0 + ref.sum(0), "colsum of the stored values")


@pytest.mark.parametrize("out_dt", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("bn", [64, 128])
def test_gelu_and_aux_out(bn, out_dt):
    """aux_out (bf16 pre-activation) exact; GELU against fp64 erf within fp32 erff error."""
    g = gen(21 + bn)
    A, B = ints(g, EM, EK) / 8, ints(g, EN, EK) / 8
    bias = ints(g, EN, r=16) / 8
    a, b = operands(A, B, False, False)
    ldd = EN + 3
    d = torch.empty(EM, ldd, device="cuda", dtype=out_dt)
    pre = torch.full((EM, ldd), 7.0, device="cuda", dtype=BF16)
    gemm(a, b, d, EM, EN, EK, bn=bn, bias=bias.float(), act=ACT_GELU, aux_out=pre)
    z = A @ B.t() + bias
    assert_exact(pre[:, :EN], z, "aux_out")
    assert bool((pre[:, EN:] == 7.0).all())
    ref = 0.5 * z * (1 + torch.special.erf(z / 2 ** 0.5))
    assert_bound(d[:, :EN], ref, 2.0 ** -20 * (1 + z.abs()), "gelu")


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("bn", [64, 128])
def test_act_bwd(bn, mode):
    """act_bwd 1: out = acc * (aux > 0), exact (zeros and -0 in aux); 2: out = acc * gelu'(aux)."""
    g = gen(31 + bn + mode)
    A, B = ints(g, EM, EK), ints(g, EN, EK)
    a, b = operands(A, B, False, True)
    ldd = EN + 1
    aux = torch.randn(EM, ldd, device="cuda", generator=g).to(BF16)
    aux[::3, ::5] = 0.0
    aux[1::3, ::7] = -0.0
    d = torch.empty(EM, ldd, device="cuda", dtype=F32)
    gemm(a, b, d, EM, EN, EK, bn=bn, b_mn=True, aux_in=aux, act_bwd=mode, alpha=-1.0)
    acc = -(A @ B.t())
    x = aux[:, :EN].double()
    if mode == 1:
        assert_exact(d[:, :EN], acc * (x > 0), "relu' mask")
    else:
        dg = 0.5 * (1 + torch.special.erf(x / 2 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5
        assert_bound(d[:, :EN], acc * dg, acc.abs() * 2.0 ** -17, "gelu' mask")


@pytest.mark.parametrize("bn", [64, 128])
def test_alpha_rounding_and_e4m3_output(bn):
    """alpha = 0.3 (not a power of two) on random-normal operands against the elementwise
    bound; e4m3 output of an exact result equals its round-to-nearest-even e4m3 value."""
    g = gen(41 + bn)
    A = torch.randn(EM, EK, device="cuda", generator=g, dtype=torch.float64).to(BF16).double()
    B = torch.randn(EN, EK, device="cuda", generator=g, dtype=torch.float64).to(BF16).double()
    a, b = operands(A, B, False, False, extra=8)
    d = torch.empty(EM, EN, device="cuda", dtype=F32)
    gemm(a, b, d, EM, EN, EK, bn=bn, alpha=0.3)
    assert_bound(d, 0.3 * (A @ B.t()), acc_bound(A, B, EK, 0.3) + 2 * U32 * (0.3 * (A @ B.t())).abs(),
                 "alpha=0.3")
    db = torch.empty(EM, EN, device="cuda", dtype=BF16)
    gemm(a, b, db, EM, EN, EK, bn=bn, alpha=0.3)
    assert_bound(db, 0.3 * (A @ B.t()), 2 * acc_bound(A, B, EK, 0.3), "alpha=0.3 bf16")
    Ai, Bi = ints(g, EM, EK), ints(g, EN, EK)
    a, b = operands(Ai, Bi, False, False)
    ldd = EN + 1
    q = torch.full((EM, ldd), 7.0, device="cuda").to(E4M3)
    gemm(a, b, q, EM, EN, EK, bn=bn, alpha=2.0 ** -6)
    ref = (Ai @ Bi.t()) * 2.0 ** -6
    assert float(ref.abs().max()) < 448
    assert_exact(q[:, :EN], ref, "e4m3 output")
    assert bool((q[:, EN:].float() == 7.0).all())


@pytest.mark.parametrize("ldd", [EN, EN + 4, EN + 3, EN + 1], ids=lambda v: f"ldd{v}")
@pytest.mark.parametrize("bn", [64, 128])
def test_accumulate(bn, ldd):
    """accumulate=True adds into fp32 d: red.add.v4 when ldd % 4 == 0, scalar atomics otherwise."""
    g = gen(51 + bn + ldd)
    A, B = ints(g, EM, EK), ints(g, EN, EK)
    bias = ints(g, EN, r=30)
    a, b = operands(A, B, True, True)
    dst = ints(g, EM + 2, ldd, r=1000)
    d = dst.float()
    gemm(a, b, d, EM, EN, EK, bn=bn, a_mn=True, b_mn=True, bias=bias.float(), accumulate=True)
    ref = dst.clone()
    ref[:EM, :EN] += A @ B.t() + bias
    assert_exact(d, ref, f"d += A B^T + bias, ldd={ldd}")


@pytest.mark.parametrize("which", ["a", "b", "both"])
@pytest.mark.parametrize("bn", [64, 128])
def test_batched_broadcast_and_bias_ptrs(bn, which):
    """Batched A and/or B (batch_stride 0 on the other side), batched D with a stride that is
    not M * ldd, per-batch bias pointers (one of them null)."""
    g = gen(61 + bn)
    nb, M, N, K = 3, 129, 130, 136
    A = ints(g, nb if which != "b" else 1, M, K)
    B = ints(g, nb if which != "a" else 1, N, K)
    a, b = operands(A, B, False, False, extra=8)
    a2, b2 = (a if which != "b" else a[0]), (b if which != "a" else b[0])
    biases = [ints(g, N, r=100).float(), None, ints(g, N, r=100).float()]
    ptrs = torch.tensor([t.data_ptr() if t is not None else 0 for t in biases], device="cuda",
                        dtype=torch.int64)
    ldd = N + 2
    dst = torch.full((nb, M + 1, ldd), 7.0, device="cuda")
    gemm(a2, b2, dst, M, N, K, bn=bn, batch=nb, a_bs=a.stride(0) if which != "b" else 0,
         b_bs=b.stride(0) if which != "a" else 0, ldd=ldd, d_bs=dst.stride(0), bias_ptrs=ptrs)
    for i in range(nb):
        ref = A[i if which != "b" else 0] @ B[i if which != "a" else 0].t()
        if biases[i] is not None:
            ref = ref + biases[i].double()
        assert_exact(dst[i, :M, :N], ref, f"batch {i}")
    assert bool((dst[:, M:, :] == 7.0).all()) and bool((dst[:, :, N:] == 7.0).all())


# -------------------------------------------------------------------------------------- split-K
@pytest.mark.parametrize("K,split", [(448, 3), (310, 4), (1000, 8), (64, 4)],
                         ids=["uneven_7kb_3", "empty_5kb_4", "even_16kb_8", "clamped_1kb_4"])
@pytest.mark.parametrize("bn", [64, 128])
def test_split_k_adds_into_d(bn, K, split):
    """Split-K into a non-zero d: d += A B^T + bias (the bias once), colsum += its column sums;
    also when splits get no K-blocks and when the split count is clamped to the K-blocks."""
    g = gen(71 + bn + K)
    A, B = ints(g, EM, K), ints(g, EN, K)
    bias = ints(g, EN, r=30)
    a, b = operands(A, B, True, True)
    d0 = ints(g, EM, EN, r=1000)
    d = d0.float()
    c0 = ints(g, EN, r=1000)
    colsum = c0.float()
    gemm(a, b, d, EM, EN, K, bn=bn, a_mn=True, b_mn=True, bias=bias.float(), colsum=colsum,
         split_k=split)
    prod = A @ B.t() + bias
    assert_exact(d, d0 + prod, "split-K sum added into d")
    assert_exact(colsum, c0 + prod.sum(0), "split-K colsum")


REJECTED = {
    "splitk_relu": dict(split_k=2, act=ACT_RELU),
    "splitk_gelu": dict(split_k=2, act=ACT_GELU),
    "splitk_aux_out": dict(split_k=2, aux_out=True),
    "splitk_act_bwd": dict(split_k=2, aux_in=True, act_bwd=1),
    "splitk_bf16_d": dict(split_k=2, out=BF16),
    "accumulate_bf16_d": dict(accumulate=True, out=BF16),
    "accumulate_e4m3_d": dict(accumulate=True, out=E4M3),
}


@pytest.mark.parametrize("case", list(REJECTED))
def test_rejected_combinations_launch_nothing(case):
    """Epilogues that cannot be right (a nonlinear epilogue on a split-K partial sum, accumulate
    into a store that overwrites) raise before any launch and leave d as it was."""
    kw = dict(REJECTED[case])
    g = gen(81)
    M, N, K = 256, 128, 512
    a, b = operands(ints(g, M, K), ints(g, N, K), False, False)
    d = torch.full((M, N), 7.0, device="cuda").to(kw.pop("out", F32))
    if kw.pop("aux_out", False):
        kw["aux_out"] = torch.zeros(M, N, device="cuda", dtype=BF16)
    if kw.pop("aux_in", False):
        kw["aux_in"] = torch.ones(M, N, device="cuda", dtype=BF16)
    n0 = launches()
    with pytest.raises(RuntimeError, match="invalid argument"):
        gemm(a, b, d, M, N, K, bn=64, **kw)
    torch.cuda.synchronize()
    assert launches() == n0
    assert bool((d.float() == 7.0).all())


# ------------------------------------------------------------------------- row-wise epilogues
XENT_CASES = [(n, pad, bn) for n in (2, 10, 32, 62, 64, 65, 100, 128) for pad in ("r8", "p8")
              for bn in ((64, 128) if n <= 64 else (128,))]


@pytest.mark.parametrize("N,pad,bn", XENT_CASES)
def test_xent(N, pad, bn):
    """Softmax-cross-entropy epilogue on exactly representable logits: loss sum against fp64
    logsumexp, dlogits elementwise, every pad column of a dlogits row zero (ldd = round_up(N, 8)
    and N + 8), rows past M untouched, #correct, colsum, alpha; some labels on the last class."""
    g = gen(91 + N + bn)
    M, K = 300, 200
    A, B = ints(g, M, K) / 8, ints(g, N, K) / 8
    bias = ints(g, N, r=16) / 8
    alpha = 0.5 if (N + bn) % 3 else 1.0
    labels = torch.randint(0, N, (M,), device="cuda", generator=g, dtype=torch.int32)
    labels[::7] = N - 1
    ldd = (N + 7) // 8 * 8 if pad == "r8" else N + 8
    dl = torch.full((M + 2, ldd), 7.0, device="cuda", dtype=BF16)
    loss = torch.zeros(1, device="cuda")
    corr = torch.full((2,), 5, device="cuda", dtype=torch.int32)
    colsum = torch.zeros(N, device="cuda")
    a, b = operands(A, B, False, False)
    gemm(a, b, dl, M, N, K, bn=bn, epi=EPI_XENT, d_dtype=1, ldd=ldd, alpha=alpha,
         bias=bias.float(), labels=labels, grad_scale=1.0 / M, loss_sum=loss, correct=corr,
         colsum=colsum)
    z = alpha * (A @ B.t()) + bias
    assert torch.equal(z.float().double(), z)          # the logits are exact in fp32
    lab = labels.long()
    lse = torch.logsumexp(z, 1)
    ref_loss = (lse - z.gather(1, lab[:, None])[:, 0]).sum()
    # per row: __expf / __logf and an N-term fp32 sum; then the fp32 reduction over the rows
    assert abs(loss.item() - ref_loss.item()) <= 2e-5 * M + 64 * U32 * abs(ref_loss.item())
    p = torch.softmax(z, 1)
    gref = (p - torch.nn.functional.one_hot(lab, N).double()) / M
    g32_bound = p * 4e-5 / M + 2.0 ** -22 * gref.abs()
    assert_bound(dl[:M, :N], gref, g32_bound, "dlogits")
    assert bool((dl[:M, N:] == 0).all()), "pad columns of dlogits rows must be zero"
    assert bool((dl[M:] == 7.0).all()), "rows past M written"
    assert int(corr[0]) == 5 + int((z.argmax(1) == lab).sum())
    assert int(corr[1]) == 5
    assert_bound(colsum, gref.sum(0), g32_bound.sum(0) + M * U32 * gref.abs().sum(0), "colsum")


@pytest.mark.parametrize("N,bn", [(10, 64), (62, 64), (64, 64), (64, 128), (65, 128), (100, 128),
                                  (128, 128)])
def test_argmax_batched_first_max_on_ties(N, bn):
    """Argmax-accuracy epilogue, batched, labels with a batch stride: on exact ties the kernel
    keeps the first maximum, as torch.argmax does (the data make first-max and last-max differ)."""
    g = gen(101 + N + bn)
    nb, M, K = 3, 300, 128
    A = ints(g, nb, M, K)
    B = ints(g, nb, N, K)
    B[:, 1::2] = B[:, 0::2][:, :N // 2]                  # column 2j + 1 duplicates column 2j
    bias = ints(g, N, r=20)
    bias[1::2] = bias[0::2][:N // 2]
    alpha = -0.5 if N % 2 else 1.0
    z = alpha * (A @ B.transpose(1, 2)) + bias
    first = z.argmax(2)
    last = N - 1 - z.flip(2).argmax(2)
    lab = last.clone()
    lab[:, ::3] = first[:, ::3]                          # a third of the rows: the first maximum
    lbs = M + 5
    labels = torch.full((nb, lbs), -1, device="cuda", dtype=torch.int32)
    labels[:, :M] = lab.int()
    want = (first == lab).sum(1)
    assert not torch.equal(want, (last == lab).sum(1)), "data must separate first- and last-max"
    a, b = operands(A, B, False, False)
    corr = torch.full((nb + 1,), 5, device="cuda", dtype=torch.int32)
    gemm(a, b, None, M, N, K, bn=bn, batch=nb, a_bs=a.stride(0), b_bs=b.stride(0), epi=EPI_ARGMAX,
         alpha=alpha, bias=bias.float(), labels=labels, labels_bs=lbs, correct=corr)
    assert corr[:nb].tolist() == (5 + want).tolist()
    assert int(corr[nb]) == 5


@pytest.mark.parametrize("epi", [EPI_XENT, EPI_ARGMAX], ids=["xent", "argmax"])
@pytest.mark.parametrize("N,bn", [(129, 128), (129, 0), (100, 64)])
def test_rowwise_wider_than_tile_rejected(epi, N, bn):
    g = gen(111)
    M, K = 128, 64
    a, b = operands(ints(g, M, K), ints(g, N, K), False, False)
    labels = torch.zeros(M, device="cuda", dtype=torch.int32)
    corr = torch.zeros(1, device="cuda", dtype=torch.int32)
    loss = torch.zeros(1, device="cuda")
    n0 = launches()
    with pytest.raises(RuntimeError):
        gemm(a, b, None, M, N, K, bn=bn, epi=epi, labels=labels, correct=corr, loss_sum=loss)
    assert launches() == n0


def test_xent_dlogits_narrower_than_a_row_rejected():
    """A dlogits stride below N would make rows overlap: refused before any launch."""
    g = gen(112)
    M, N, K = 128, 62, 64
    a, b = operands(ints(g, M, K), ints(g, N, K), False, False)
    dl = torch.full((M, 56), 7.0, device="cuda", dtype=BF16)
    labels = torch.zeros(M, device="cuda", dtype=torch.int32)
    loss = torch.zeros(1, device="cuda")
    n0 = launches()
    with pytest.raises(RuntimeError, match="invalid argument"):
        gemm(a, b, dl, M, N, K, bn=64, epi=EPI_XENT, d_dtype=1, labels=labels, loss_sum=loss)
    assert launches() == n0 and bool((dl == 7.0).all())


# -------------------------------------------------------------------------------- e4m3 inputs
@pytest.mark.parametrize("M,N,K,nb", [(1, 8, 16, 1), (129, 65, 144, 1), (300, 200, 528, 1),
                                      (128, 64, 16, 1), (130, 70, 528, 3), (257, 130, 144, 2)])
def test_fp8_inputs_exact(M, N, K, nb):
    """e4m3 K-major operands (widened to f16 per stage, fp32 accumulation): exact, with tails in
    M, N and K (the 3-stage ring wraps at K = 528), batched."""
    g = gen(121 + M + K)
    A, B = ints(g, nb, M, K), ints(g, nb, N, K)
    a, b = operands(A, B, False, False, dtype=E4M3, extra=16 * (K % 3 == 0))
    ldd = N + 1
    d = torch.full((nb, M, ldd), 7.0, device="cuda")
    if nb == 1:
        gemm(a[0], b[0], d[0], M, N, K, bn=64)
    else:
        gemm(a, b, d, M, N, K, bn=64, batch=nb, a_bs=a.stride(0), b_bs=b.stride(0), d_bs=d.stride(0))
    for i in range(nb):
        assert_exact(d[i, :, :N], A[i] @ B[i].t(), f"fp8 batch {i}")
    assert bool((d[:, :, N:] == 7.0).all())


@pytest.mark.parametrize("layout", ["t01", "t10", "t11"])
def test_fp8_mn_major_rejected(layout):
    a_mn, b_mn = LAYOUTS[layout]
    g = gen(131)
    a, b = operands(ints(g, 128, 128), ints(g, 64, 128), a_mn, b_mn, dtype=E4M3)
    d = torch.zeros(128, 64, device="cuda")
    n0 = launches()
    with pytest.raises(RuntimeError, match="not supported"):
        gemm(a, b, d, 128, 64, 128, bn=64, a_mn=a_mn, b_mn=b_mn)
    assert launches() == n0


# -------------------------------------------------------------- peer-table (committee) form
def gemm_dynamic_layout(kmax):
    """Field offsets of ``GemmDynamic`` (bflc_kernels.h) under natural alignment."""
    fields = [("active_batches", 4, 1), ("map_index", 4, kmax), ("bias", 8, kmax),
              ("wait_flag", 8, kmax), ("wait_value", 4, 1)]
    off, o, align = {}, 0, 1
    for name, size, count in fields:
        o = (o + size - 1) // size * size
        off[name] = o
        o += size * count
        align = max(align, size)
    return off, (o + align - 1) // align * align


def gemm_dynamic(active, map_index, bias_ptrs):
    """A device-resident GemmDynamic with every wait_flag null."""
    sz = C().struct_sizes()
    kmax = sz["kMaxRanks"]
    off, size = gemm_dynamic_layout(kmax)
    assert size == sz["GemmDynamic"]
    buf = bytearray(size)
    struct.pack_into("<i", buf, off["active_batches"], active)
    struct.pack_into(f"<{kmax}i", buf, off["map_index"], *(list(map_index) + [0] * (kmax - len(map_index))))
    struct.pack_into(f"<{kmax}Q", buf, off["bias"], *(list(bias_ptrs) + [0] * (kmax - len(bias_ptrs))))
    return torch.frombuffer(buf, dtype=torch.uint8).cuda()


@pytest.mark.parametrize("bn", [64, 128])
def test_peer_table_committee_form(bn):
    """The committee's two validation GEMMs: B from a device table of tensor maps (one per
    distinct weight allocation, box = the forced BN), a GemmDynamic choosing map and bias per
    batch (a permuted map_index, one null bias) and active_batches < batch.  Batches past
    active_batches leave their d slice and correct[b] untouched."""
    kmax = C().struct_sizes()["kMaxRanks"]
    g = gen(141 + bn)
    nb, active, M, K, H = 4, 3, 300, 200, 200
    NC = 62 if bn == 64 else 100
    W1 = [padded(ints(g, H, K), BF16) for _ in range(nb)]
    W2 = [padded(ints(g, NC, H), BF16) for _ in range(nb)]
    maps = bytearray(2 * kmax * 128)
    for i in range(nb):
        maps[i * 128:(i + 1) * 128] = C().gemm_b_map(W1[i].data_ptr(), H, K, W1[i].stride(0), False,
                                                     False, EPI_GENERIC, bn)
        j = kmax + i
        maps[j * 128:(j + 1) * 128] = C().gemm_b_map(W2[i].data_ptr(), NC, H, W2[i].stride(0), False,
                                                     False, EPI_ARGMAX, bn)
    b_maps = torch.frombuffer(maps, dtype=torch.uint8).cuda()
    perm = [2, 0, 3, 1]
    b1 = [ints(g, H, r=100).float() if i != 1 else None for i in range(nb)]
    b2 = [ints(g, NC, r=100).float() for _ in range(nb)]
    dyn1 = gemm_dynamic(active, perm, [t.data_ptr() if t is not None else 0 for t in b1])
    dyn2 = gemm_dynamic(active, [kmax + p for p in perm], [t.data_ptr() for t in b2])

    X = ints(g, M, K)
    x = padded(X, BF16)
    h = torch.full((nb, M, H), 7.0, device="cuda", dtype=BF16)
    gemm(x, W1[0], h, M, H, K, bn=bn, batch=nb, ldd=H, d_bs=M * H, act=ACT_RELU, b_maps=b_maps,
         dyn_ptr=dyn1.data_ptr())
    X2 = ints(g, nb, M, H)
    x2 = padded(X2, BF16)
    labels = torch.randint(0, NC, (M,), device="cuda", generator=g, dtype=torch.int32)
    corr = torch.full((nb,), 1000, device="cuda", dtype=torch.int32)
    gemm(x2, W2[0], None, M, NC, H, bn=bn, batch=nb, a_bs=x2.stride(0), epi=EPI_ARGMAX, labels=labels,
         correct=corr, b_maps=b_maps, dyn_ptr=dyn2.data_ptr())
    for i in range(nb):
        if i >= active:
            assert bool((h[i] == 7.0).all()), f"inactive batch {i} wrote d"
            assert int(corr[i]) == 1000, f"inactive batch {i} counted"
            continue
        w = perm[i]
        z1 = X @ W1[w].double().t() + (b1[i].double() if b1[i] is not None else 0)
        assert_exact(h[i], torch.relu(z1), f"layer 1 batch {i} (map {w})")
        z2 = X2[i] @ W2[w].double().t() + b2[i].double()
        assert int(corr[i]) == 1000 + int((z2.argmax(1) == labels.long()).sum()), f"batch {i}"


# ------------------------------------------------------------------------------------- gemm2
GEMM2_CASES = [
    # M, N, K, out dtype, alpha, bias, act, exact operands
    (4096, 4096, 256, F32, 1.0, False, ACT_NONE, True),
    (8192, 3072, 768, BF16, 0.5, True, ACT_RELU, True),
    (4096, 4096, 256, BF16, 1.0, True, ACT_GELU, False),
    (612, 520, 8, F32, 1.0, True, ACT_GELU, False),
    (612, 520, 100, BF16, 0.25, True, ACT_RELU, True),
    (612, 520, 100, F32, -0.5, False, ACT_NONE, True),
]


@pytest.mark.parametrize("M,N,K,out_dt,alpha,use_bias,act,exact", GEMM2_CASES,
                         ids=[f"{c[0]}x{c[1]}x{c[2]}-{'f32' if c[3] == F32 else 'bf16'}-act{c[6]}"
                              for c in GEMM2_CASES])
def test_gemm2(M, N, K, out_dt, alpha, use_bias, act, exact):
    """CTA-pair kernel: tile counts past one wave of resident clusters (the persistent tile loop
    carries ring stage and phase across tiles), M = 612 (the last cluster's rank-1 CTA has no
    row inside M), N = 520 (8 valid columns in the last tile), K of one and two K-blocks."""
    g = gen(151 + M + K)
    s = 1.0 if exact else 1.0 / 8
    A, B = ints(g, M, K) * s, ints(g, N, K) * s
    bias = ints(g, N, r=64) / (1 if exact else 8) if use_bias else None
    a, b = operands(A, B, False, False)
    ldd = N + 4
    dst = torch.full((M + 8, ldd), 7.0, device="cuda", dtype=out_dt)
    C().gemm2(a, b, dst, M, N, K, a.stride(0), b.stride(0), alpha,
              bias.float() if bias is not None else None, act)
    z = alpha * (A @ B.t()) + (bias if bias is not None else 0)
    if act == ACT_RELU:
        z = torch.relu(z)
    if act == ACT_GELU:
        ref = 0.5 * z * (1 + torch.special.erf(z / 2 ** 0.5))
        assert_bound(dst[:M, :N], ref, 2.0 ** -20 * (1 + z.abs()), "gemm2 gelu")
    else:
        assert_exact(dst[:M, :N], z, "gemm2")
    assert bool((dst[M:] == 7.0).all()) and bool((dst[:, N:] == 7.0).all())


@pytest.mark.parametrize("out_dt", [F32, BF16], ids=["f32", "bf16"])
def test_ops_gemm_routes_big_problems_to_gemm2(monkeypatch, out_dt):
    """``ops.gemm.gemm`` sends a big plain K-major problem to gemm2 and its result equals the
    same problem forced through gemm_sm100.  A counting shim on the native ``gemm2`` tells the
    two apart (both kernels bump launch_count)."""
    from bflc_demo_b200.ops import gemm as G
    m = C()
    calls = []
    orig = m.gemm2

    def counting(*args, **kw):
        calls.append(args[3:6])
        return orig(*args, **kw)

    monkeypatch.setattr(m, "gemm2", counting)
    g = gen(161)
    M, N, K = 2048, 2048, 320
    A, B = ints(g, M, K), ints(g, N, K)
    bias = ints(g, N, r=64)
    a, b = A.to(BF16), B.to(BF16)
    d2 = G.gemm(a, b, out_dtype=out_dt, alpha=0.5, bias=bias.float(), act=G.ACT_RELU)
    assert calls == [(M, N, K)]
    monkeypatch.setattr(G, "_GEMM2", False)
    d1 = G.gemm(a, b, out_dtype=out_dt, alpha=0.5, bias=bias.float(), act=G.ACT_RELU)
    assert len(calls) == 1
    assert torch.equal(d1, d2)
    assert_exact(d2, torch.relu(0.5 * (A @ B.t()) + bias), "ops.gemm")
