"""The wgmma GEMM's low-rank K tail (``csrc/kernels/gemm_sm100.cu``, ``gemm_tail_kernel``):
``D = alpha * (A.B^T + A2.B2^T)`` through the generic epilogues, in the two forms a LoRA linear uses

* forward        -- A = x [M, K], B = W [N, K] K-major; A2 = u [M, r], B2 = the adapter B [N, r];
* input gradient -- A = dz [M, K], B = W read MN-major ([K, N]); A2 = v [M, r], B2 = the adapter
                    A read MN-major ([r, N]).

Exact cases use small-integer operands (every partial sum exact in fp32), so an fp32 result equals
the fp64 product bit for bit and a bf16 one equals it rounded once; random cases are held to the
fp32-accumulation bound.  Every output sits in a NaN-filled frame that must survive.  Needs an H100.
"""
import pytest
import torch

from bflc_demo_b200._native import C
from bflc_demo_b200.ops import gemm as G

pytestmark = pytest.mark.gpu

BF16, F32 = torch.bfloat16, torch.float32
DT = {F32: 0, BF16: 1}
U32 = 2.0 ** -24
HALF_ULP = {F32: 2.0 ** -24, BF16: 2.0 ** -8}
RANKS = (8, 16, 32, 64)


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def ints(g, *shape, r=4):
    return torch.randint(-r, r + 1, shape, generator=g, device="cuda").double()


def framed(M, N, dtype, pad=8):
    """A NaN-filled [M + 2, N + pad (rounded to 8)] buffer and the [M, N] view at row 1 inside it."""
    ld = (N + pad + 7) // 8 * 8
    buf = torch.full((M + 2, ld), float("nan"), device="cuda", dtype=dtype)
    return buf, buf[1:M + 1, :N]


def frame_intact(buf, M, N):
    outside = torch.ones_like(buf, dtype=torch.bool)
    outside[1:M + 1, :N] = False
    return bool(torch.isnan(buf[outside].float()).all())


def tail_gemm(a, b, a2, b2, d, M, N, K, *, bn, b_mn=False, alpha=1.0, bias=None, act=0, aux_out=None):
    r = a2.shape[1]
    C().gemm(a, b, d, M, N, K, 1, a.stride(0), b.stride(0), 0, 0, False, b_mn, False, 0, DT[d.dtype],
             d.stride(0), 0, alpha, bias, act, aux_out, None, 0, None, 1, False, None, 0, 1.0, None, None,
             None, None, 0, 0, 0, 0, 0, bn, a2, b2, r)


def operands(form, A, B, A2, B2):
    """Device bf16 operands of the logical A [M,K], B [N,K], A2 [M,r], B2 [N,r] in ``form``."""
    if form == "fwd":
        return A.to(BF16), B.to(BF16).contiguous(), A2.to(BF16), B2.to(BF16).contiguous(), False
    return (A.to(BF16), B.t().contiguous().to(BF16), A2.to(BF16), B2.t().contiguous().to(BF16), True)


SHAPES = [(200, 136, 200), (128, 64, 64), (77, 264, 392)]


@pytest.mark.parametrize("form", ["fwd", "dx"])
@pytest.mark.parametrize("r", RANKS)
@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_tail_exact(form, r, bn, shape):
    M, N, K = shape
    g = gen(r * 1000 + bn + M)
    A, B, A2, B2 = ints(g, M, K), ints(g, N, K), ints(g, M, r), ints(g, N, r)
    bias = ints(g, N).float()
    a, b, a2, b2, b_mn = operands(form, A, B, A2, B2)
    ref = A @ B.T + A2 @ B2.T
    # fp32 out, alpha 0.5, no activation
    buf, d = framed(M, N, F32)
    tail_gemm(a, b, a2, b2, d, M, N, K, bn=bn, b_mn=b_mn, alpha=0.5)
    torch.cuda.synchronize()
    assert torch.equal(d.double(), 0.5 * ref)
    assert frame_intact(buf, M, N)
    # bf16 out, bias + ReLU
    buf, d = framed(M, N, BF16)
    tail_gemm(a, b, a2, b2, d, M, N, K, bn=bn, b_mn=b_mn, bias=bias, act=G.ACT_RELU)
    want = (ref + bias.double()).clamp_min(0).float().to(BF16)
    assert torch.equal(d, want)
    assert frame_intact(buf, M, N)
    # bf16 out, bias + GELU with the pre-activation copy
    buf, d = framed(M, N, BF16)
    abuf, aux = framed(M, N, BF16)
    assert aux.stride(0) == d.stride(0)
    tail_gemm(a, b, a2, b2, d, M, N, K, bn=bn, b_mn=b_mn, bias=bias, act=G.ACT_GELU, aux_out=aux)
    pre = ref + bias.double()
    assert torch.equal(aux, pre.float().to(BF16))
    gelu = torch.nn.functional.gelu(pre)
    tol = 2.0 ** -8 * gelu.abs() + 1e-3 * pre.abs().clamp_min(1.0)
    assert bool(((d.double() - gelu).abs() <= tol).all())
    assert frame_intact(buf, M, N) and frame_intact(abuf, M, N)


@pytest.mark.parametrize("form", ["fwd", "dx"])
@pytest.mark.parametrize("r", RANKS)
@pytest.mark.parametrize("bn", [64, 128])
def test_tail_random_within_fp32_bound(form, r, bn):
    M, N, K = 384, 200, 768
    g = gen(7 * r + bn)
    A, B = torch.randn(M, K, generator=g, device="cuda"), torch.randn(N, K, generator=g, device="cuda")
    A2, B2 = torch.randn(M, r, generator=g, device="cuda"), torch.randn(N, r, generator=g, device="cuda")
    A, B, A2, B2 = (t.to(BF16).double() for t in (A, B, A2, B2))
    a, b, a2, b2, b_mn = operands(form, A, B, A2, B2)
    buf, d = framed(M, N, F32)
    tail_gemm(a, b, a2, b2, d, M, N, K, bn=bn, b_mn=b_mn)
    ref = A @ B.T + A2 @ B2.T
    bound = 2.0 * (K + r) * U32 * (A.abs() @ B.abs().T + A2.abs() @ B2.abs().T) + 2.0 ** -126
    assert bool(((d.double() - ref).abs() <= bound).all())
    assert frame_intact(buf, M, N)


@pytest.mark.parametrize("form", ["fwd", "dx"])
@pytest.mark.parametrize("bn", [64, 128])
def test_zero_tail_is_the_plain_gemm(form, bn):
    """With B2 = 0 the tail adds exact zeros: bit-identical to the same GEMM without a tail."""
    M, N, K, r = 300, 264, 520, 16
    g = gen(11 + bn)
    A, B = torch.randn(M, K, generator=g, device="cuda").double(), torch.randn(N, K, generator=g, device="cuda").double()
    A2 = torch.randn(M, r, generator=g, device="cuda").double()
    a, b, a2, b2, b_mn = operands(form, A, B, A2, torch.zeros(N, r, device="cuda", dtype=torch.float64))
    bias = torch.randn(N, generator=g, device="cuda")
    for dt in (F32, BF16):
        d0 = torch.empty(M, N, device="cuda", dtype=dt)
        d1 = torch.empty_like(d0)
        C().gemm(a, b, d0, M, N, K, 1, a.stride(0), b.stride(0), 0, 0, False, b_mn, False, 0, DT[dt], N, 0,
                 1.0, bias, G.ACT_GELU, None, None, 0, None, 1, False, None, 0, 1.0, None, None, None, None,
                 0, 0, 0, 0, 0, bn)
        tail_gemm(a, b, a2, b2, d1, M, N, K, bn=bn, b_mn=b_mn, bias=bias, act=G.ACT_GELU)
        assert torch.equal(d0, d1)


def test_ops_gemm_tail_at_a_large_shape():
    """ops.gemm(tail=) at a BERT FFN shape (where a plain GEMM would take the CTA-pair kernel)."""
    M, N, K, r = 2048, 3072, 768, 16
    g = gen(5)
    x = (torch.randn(M, K, generator=g, device="cuda") * 0.5).to(BF16)
    w = (torch.randn(N, K, generator=g, device="cuda") * 0.05).to(BF16)
    u = torch.randn(M, r, generator=g, device="cuda").to(BF16)
    bl = torch.randn(N, r, generator=g, device="cuda").to(BF16)
    y = G.gemm(x, w, out_dtype=F32, tail=(u, bl))
    ref = x.double() @ w.double().T + u.double() @ bl.double().T
    bound = 2.0 * (K + r) * U32 * (x.double().abs() @ w.double().abs().T + u.double().abs() @ bl.double().abs().T)
    assert bool(((y.double() - ref).abs() <= bound + 2.0 ** -126).all())


def _refusal_cases():
    M, N, K, r = 128, 128, 128, 16
    dev = "cuda"

    def t(*s, dt=BF16):
        return torch.ones(*s, device=dev, dtype=dt)

    a, b, d = t(M, K), t(N, K), torch.empty(M, N, device=dev, dtype=F32)
    a2, b2 = t(M, r), t(N, r)
    base = dict(a=a, b=b, d=d, M=M, N=N, K=K, batch=1, b_mn=False, fp8=False, epi=0, split_k=1, acc=False,
                b_maps=None, dyn=0, a2=a2, b2=b2, k2=r, a_mn=False)
    flat = t(M * r + 8)
    cases = {
        "rank_4": dict(a2=t(M, 4), b2=t(N, 4), k2=4),
        "rank_72": dict(a2=t(M, 72), b2=t(N, 72), k2=72),
        "rank_12": dict(a2=t(M, 12), b2=t(N, 12), k2=12),
        "rank_mismatch": dict(b2=t(N, 8)),
        "missing_b2": dict(b2=None),
        "a2_fp32": dict(a2=t(M, r, dt=F32)),
        "a2_shape": dict(a2=t(M + 1, r)),
        "a2_noncontig": dict(a2=t(M, 2 * r)[:, :r]),
        "a2_misaligned": dict(a2=flat[1:1 + M * r].view(M, r)),
        "a2_cpu": dict(a2=torch.ones(M, r, dtype=BF16)),
        "split_k": dict(split_k=2),
        "accumulate": dict(acc=True),
        "xent_epilogue": dict(epi=1),
        "argmax_epilogue": dict(epi=2),
        "batch_2": dict(batch=2),
        "b_maps": dict(b_maps=torch.zeros(128, device=dev, dtype=torch.uint8)),
        "a_mn": dict(a_mn=True),
        "fp8": dict(a=t(M, K).to(torch.float8_e4m3fn), b=t(N, K).to(torch.float8_e4m3fn), fp8=True),
    }
    return base, cases


REFUSALS = ["rank_4", "rank_72", "rank_12", "rank_mismatch", "missing_b2", "a2_fp32", "a2_shape", "a2_noncontig",
            "a2_misaligned", "a2_cpu", "split_k", "accumulate", "xent_epilogue", "argmax_epilogue", "batch_2",
            "b_maps", "a_mn", "fp8"]


@pytest.mark.parametrize("case", REFUSALS)
def test_tail_refusals_raise_before_launch(case):
    base, cases = _refusal_cases()
    assert sorted(cases) == sorted(REFUSALS)
    p = {**base, **cases[case]}
    before = C().launch_count()
    with pytest.raises(RuntimeError):
        C().gemm(p["a"], p["b"], p["d"], p["M"], p["N"], p["K"], p["batch"], p["K"], p["K"], 0, 0, p["a_mn"],
                 p["b_mn"], p["fp8"], p["epi"], 0, p["N"], 0, 1.0, None, 0, None, None, 0, None, p["split_k"],
                 p["acc"], None, 0, 1.0, None, None, p["b_maps"], None, 0, 0, 0, 0, p["dyn"], 0,
                 p["a2"], p["b2"], p["k2"])
    assert C().launch_count() == before


def test_ops_gemm_refuses_mismatched_tail_ranks():
    a, b = torch.ones(64, 64, device="cuda", dtype=BF16), torch.ones(64, 64, device="cuda", dtype=BF16)
    with pytest.raises(ValueError):
        G.gemm(a, b, tail=(torch.ones(64, 8, device="cuda", dtype=BF16), torch.ones(64, 16, device="cuda", dtype=BF16)))
