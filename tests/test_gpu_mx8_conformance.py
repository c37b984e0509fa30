"""MXFP8 conformance: every quantiser entry point bit for bit against the exact specification
(``ops/mx8.py::quantize_mx8_reference``), and ``gemm_mx8`` against fp64, element by element.

* CPU: ``gemm_mx8_kernel<64>`` and the three ``k_quantize_mx8`` instantiations compile with no
  stack frame and no spills.
* Quantisers (``quantize_mx8`` f32 / bf16 / u8, ``prep_inputs`` with and without the predicate,
  ``prep_inputs_chunks``, ``quantize_mlp_blob``) and ``mx8_dequant``: every e4m3 byte, every scale
  byte of the chunk array (padding rows and groups included) and the dequantised bf16, on binade
  boundaries, the clamp-to-3 and byte-247 groups, fp32 / bf16 subnormals, the saturation band,
  ties at every e4m3 binade, signed zeros, all-zero groups and every K tail.  Canary bytes around
  every output (past K rounded to 16 in a wider row pitch, rows >= R, past the scale array) must
  survive; a NaN / inf group may not disturb any other group.
* ``gemm_mx8`` on exact fixtures (``test_mx8_spec_host.exact_fixture``: small-integer codes,
  per-(row, group) scale bytes near 127, dyadic biases, power-of-two alpha): fp32 output equals
  the fp64 product bit for bit, bf16 output equals it rounded once.  Operand pad bytes are e4m3
  NaN and the output is a slice of a NaN-canaried buffer.
* ``gemm_mx8`` on quantised random normals with GELU and non-power-of-two alpha, within a bound
  derived from the kernel's rounding points; scale products outside the fp32 range.
* ``ops.nn.linear`` under ``set_precision("mx8")`` takes ``gemm_mx8`` exactly when it should and
  equals the direct calls bit for bit.
"""
import math
import os
import re
import shutil
import subprocess

import pytest
import torch

from bflc_demo_b200 import build
from bflc_demo_b200.ops.mx8 import MX8, encode_mx8, quantize_mx8_reference
from test_mx8_spec_host import exact_fixture, exact_operand, reference_out, scale_rows

U = 2.0 ** -23            # fp32 unit roundoff, doubled: allows a truncating tensor-core sum
C_CANARY, SF_CANARY = 0xAB, 0xCD


# ------------------------------------------------------------------ compilation
def test_gemm_and_quantiser_spill_free(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("no nvcc")
    inc = [f"-I{build.CSRC / d}" for d in ("include", "ledger", "runtime")]
    src = build.CSRC / "kernels" / "gemm_mx8_sm100.cu"
    proc = subprocess.run([nvcc, *build.GENCODE, *build.NVCC_FLAGS, "-Xptxas", "-v", *inc, "-c", str(src),
                           "-o", str(tmp_path / "g.o")], capture_output=True, text=True, timeout=900)
    log = proc.stdout + proc.stderr
    assert proc.returncode == 0, log[-3000:]
    props = re.findall(r"Function properties for (\w+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    found = {n: tuple(map(int, r)) for n, *r in props if "gemm_mx8_kernel" in n or "k_quantize_mx8" in n}
    assert len(found) == 4, log[-3000:]
    for name, v in found.items():
        assert v == (0, 0, 0), f"{name}: {v}"


gpu = pytest.mark.gpu


def Cm():
    from bflc_demo_b200._native import C
    return C()


# ------------------------------------------------------------------ quantiser inputs
def special_rows(K, seed):
    """Rows of groups at the edges of the rule (fp32); every row has K columns."""
    g = torch.Generator().manual_seed(seed)
    f = torch.finfo(torch.float32)
    rows = []

    def row(vals):
        r = torch.randn(K, generator=g)
        v = torch.tensor(vals, dtype=torch.float32)
        r[: min(K, v.numel())] = v[: min(K, v.numel())]
        rows.append(r)
    for k in (-118, -60, -1, 0, 1, 30, 100):                   # amax at / 1-3 ulps around 448 * 2^k
        c = torch.tensor(448.0 * 2.0 ** k, dtype=torch.float32)
        bits = c.view(torch.int32)
        for d in (-3, -2, -1, 0, 1, 2, 3):
            a = (bits + d).view(torch.float32)
            row([float(a), -float(a) / 3, float(a) / 7] * 11)
    row([2.0 ** -126, -(2.0 ** -125)] * 16)                    # clamp to byte 3
    row([f.max, -f.max / 2] * 16)                              # byte 247
    row([1e-40, -1e-41, 2.0 ** -149, -0.0] * 8)                # fp32 subnormals: flushed, all-zero
    row([448.0, 450.0, 456.0, -460.0, 463.9, 1.0] * 6)         # saturation band
    ties = []
    for b in range(-9, 9):                                     # ties to even at every e4m3 binade
        step = 2.0 ** (max(b, -6) - 3)
        ties += [2.0 ** b + step / 2, 2.0 ** b + 1.5 * step]
    row([448.0] + ties)
    row([0.0, -0.0] * 16)                                      # signed zeros, all-zero group
    row([-0.0] * 31 + [1.0])
    return torch.stack(rows)


def special_matrix(R, K, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(R, K, generator=g) * torch.logspace(-6, 6, K)
    s = special_rows(K, seed)
    n = min(R, s.shape[0])
    x[:n] = s[:n]
    return x


def canaried_q(R, K, extra_pitch):
    ld = (K + 15) // 16 * 16 + extra_pitch
    buf = torch.full((R + 3, ld), C_CANARY, dtype=torch.uint8, device="cuda")
    return buf, buf[:R]


def check_q_and_sf(qbuf, sfbuf, ref, R, K, skip_groups=()):
    w = (K + 15) // 16 * 16
    got = qbuf[:R, :w].cpu()
    want = ref.q.view(torch.uint8)
    mask = torch.ones(R, w, dtype=torch.bool)
    for r, grp in skip_groups:
        mask[r, grp * 32:(grp + 1) * 32] = False
    assert torch.equal(got[mask], want[mask])
    assert bool((qbuf[:R, w:] == C_CANARY).all()) and bool((qbuf[R:] == C_CANARY).all())
    n = ref.sf.numel()
    gs, ws = scale_rows(sfbuf[:n].cpu(), R, K), scale_rows(ref.sf, R, K)
    smask = torch.ones_like(gs, dtype=torch.bool)
    for r, grp in skip_groups:
        smask[r, grp] = False
    assert torch.equal(gs[smask], ws[smask])
    rb = (R + 255) // 256 * 256
    all_g, all_w = scale_rows(sfbuf[:n].cpu(), rb, K), scale_rows(ref.sf, rb, K)
    assert torch.equal(all_g[R:], all_w[R:])                   # padding rows: 0x7F
    assert bool((sfbuf[n:] == SF_CANARY).all())


KS = [16, 32, 48, 100, 112, 128, 784, 1000] + list(range(17, 32))     # last-group widths 16..32
RS = [1, 127, 128, 129, 255, 256, 300, 513]


@gpu
@pytest.mark.parametrize("dtype", ["f32", "bf16", "u8"])
@pytest.mark.parametrize("K", KS)
def test_quantize_mx8_bytes(dtype, K):
    from bflc_demo_b200.ops.mx8 import quantize_mx8
    for R in (RS if K in (100, 128, 784) else [129, 300]):
        for extra in (0, 32):
            x = special_matrix(R, K, seed=K + R)
            in_scale = 1.0
            if dtype == "bf16":
                x = x.clamp(-3e38, 3e38).bfloat16()
                x[0, :4] = torch.tensor([1e-39, -1e-40, 2.0 ** -133, 1.0]).bfloat16()   # bf16 subnormals
            elif dtype == "u8":
                x = torch.randint(0, 256, (R, K), generator=torch.Generator().manual_seed(K), dtype=torch.uint8)
                x[: R // 2, :32] = 0
                in_scale = 1.0 / 255.0
            ref = quantize_mx8_reference(x, in_scale=in_scale)
            qbuf, q = canaried_q(R, K, extra)
            sfbuf = torch.full((Cm().mx8_sf_bytes(R, K) + 64,), SF_CANARY, dtype=torch.uint8, device="cuda")
            out = quantize_mx8(x.cuda(), in_scale=in_scale, out=MX8(q.view(torch.float8_e4m3fn), sfbuf, R, K))
            torch.cuda.synchronize()
            check_q_and_sf(qbuf, sfbuf, ref, R, K)
            dq = torch.empty(R, (K + 15) // 16 * 16, dtype=torch.bfloat16, device="cuda")
            if extra == 0 and K % 16 == 0:
                Cm().mx8_dequant(q.contiguous(), sfbuf, dq)
                assert torch.equal(dq[:, :K].float().cpu(), ref.dequantize())


@gpu
def test_nan_group_is_isolated():
    from bflc_demo_b200.ops.mx8 import quantize_mx8
    R, K = 129, 100
    x = special_matrix(R, K, 3)
    x[5, 40] = float("nan")
    x[7, 70] = float("inf")
    clean = x.clone()
    clean[5, 32:64] = 0
    clean[7, 64:96] = 0
    ref = quantize_mx8_reference(clean)
    qbuf, q = canaried_q(R, K, 0)
    sfbuf = torch.full((Cm().mx8_sf_bytes(R, K) + 64,), SF_CANARY, dtype=torch.uint8, device="cuda")
    quantize_mx8(x.cuda(), out=MX8(q.view(torch.float8_e4m3fn), sfbuf, R, K))
    torch.cuda.synchronize()
    check_q_and_sf(qbuf, sfbuf, ref, R, K, skip_groups=[(5, 1), (7, 2)])


def _prep_outputs(R, K):
    sfn = Cm().mx8_sf_bytes(R, K)
    return (torch.full((R, K), -7.0, dtype=torch.bfloat16, device="cuda"),
            torch.full((R + 3, K), C_CANARY, dtype=torch.uint8, device="cuda"),
            torch.full((sfn + 64,), SF_CANARY, dtype=torch.uint8, device="cuda"),
            torch.full((R, K), -7.0, dtype=torch.bfloat16, device="cuda"))


def _check_prep(x, outs, R, K):
    xb, q, sf, dq = outs
    scale = 1.0 / 255.0
    ref = quantize_mx8_reference(x, in_scale=scale)
    assert torch.equal(xb.cpu(), (x.float() * scale).bfloat16())
    assert torch.equal(q[:R].cpu(), ref.q.view(torch.uint8)[:, :K]) and bool((q[R:] == C_CANARY).all())
    n = ref.sf.numel()
    gs, ws = scale_rows(sf[:n].cpu(), (R + 255) // 256 * 256, K), scale_rows(ref.sf, (R + 255) // 256 * 256, K)
    G = (K + 31) // 32
    assert torch.equal(gs[:R, :G], ws[:R, :G])
    assert bool((gs[R:] == SF_CANARY).all()) and bool((gs[:, G:] == SF_CANARY).all())   # never written
    assert bool((sf[n:] == SF_CANARY).all())
    assert torch.equal(dq.float().cpu(), ref.dequantize())


@gpu
@pytest.mark.parametrize("R,K", [(1, 16), (129, 48), (300, 784), (256, 112), (127, 1008)])
def test_prep_inputs_and_chunks(R, K):
    g = torch.Generator().manual_seed(R * K)
    x = torch.randint(0, 256, (R, K), generator=g, dtype=torch.uint8)
    x[: R // 3, : K // 2] = torch.randint(0, 3, (R // 3, K // 2), generator=g, dtype=torch.uint8)
    x[R // 2:, :16] = 0
    xc = x.cuda()
    outs = _prep_outputs(R, K)
    xb, q, sf, dq = outs
    # predicate off: nothing is written
    pred = torch.zeros(1, dtype=torch.int32, device="cuda")
    Cm().set_predicate(pred.data_ptr())
    try:
        Cm().prep_inputs(xc, xb, q[:R], sf, 1.0 / 255.0, dq)
        torch.cuda.synchronize()
    finally:
        Cm().set_predicate(0)
    assert bool((q == C_CANARY).all()) and bool((sf == SF_CANARY).all()) and bool((dq == -7.0).all())
    Cm().prep_inputs(xc, xb, q[:R], sf, 1.0 / 255.0, dq)
    torch.cuda.synchronize()
    _check_prep(x, outs, R, K)
    for steps in (1, 3) if R % 3 == 0 else (1,):
        outs = _prep_outputs(R, K)
        xb, q, sf, dq = outs
        flags = torch.ones(16, device="cuda", dtype=torch.int32)
        seq = torch.zeros(1, device="cuda", dtype=torch.int32)
        cnt = torch.zeros(16, device="cuda", dtype=torch.int32)
        ready = torch.zeros(16, device="cuda", dtype=torch.int32)
        err = torch.zeros(1, device="cuda", dtype=torch.int32)
        Cm().prep_inputs_chunks(xc, xb, q[:R], sf, R // steps, steps, 1.0 / 255.0, flags, seq, cnt, ready, err, dq)
        torch.cuda.synchronize()
        assert int(err.item()) == 0 and ready[:steps].tolist() == [1] * steps
        _check_prep(x, outs, R, K)


@gpu
@pytest.mark.parametrize("in_dim,hidden,ncls", [(784, 256, 62), (100, 128, 10), (1000, 300, 64)])
def test_quantize_mlp_blob(in_dim, hidden, ncls):
    L = Cm().mx8_mlp_layout(in_dim, hidden)
    n1, n2 = hidden * in_dim, ncls * hidden
    master = torch.zeros(n1 + hidden + n2 + ncls)
    master[:n1] = special_matrix(hidden, in_dim, 1).clamp(-1e30, 1e30).reshape(-1)
    master[n1:n1 + hidden] = torch.randn(hidden)
    master[n1 + hidden:n1 + hidden + n2] = special_matrix(ncls, hidden, 2).clamp(-1e30, 1e30).reshape(-1)
    master[n1 + hidden + n2:] = torch.randn(ncls)
    blob = torch.full((L["total"] + 64,), C_CANARY, dtype=torch.uint8, device="cuda")
    dq = torch.full((n1 + 64 * hidden,), -7.0, dtype=torch.bfloat16, device="cuda")
    Cm().quantize_mlp_blob(master.cuda(), [0, n1, n1 + hidden, n1 + hidden + n2], in_dim, hidden, ncls, blob, dq)
    torch.cuda.synchronize()
    b = blob.cpu()
    w1 = master[:n1].view(hidden, in_dim)
    w2 = torch.zeros(64, hidden)
    w2[:ncls] = master[n1 + hidden:n1 + hidden + n2].view(ncls, hidden)
    for w, R, K, qo, so, kb, rb, off in ((w1, hidden, in_dim, L["w1q"], L["w1sf"], L["kb1"], (hidden + 127) // 128, 0),
                                         (w2, 64, hidden, L["w2q"], L["w2sf"], L["kb2"], 1, n1)):
        ref = quantize_mx8_reference(w)
        assert torch.equal(b[qo:qo + R * K].view(R, K), ref.q.view(torch.uint8)[:, :K])
        sf = b[so:so + rb * kb * 512]
        want = scale_rows(ref.sf, rb * 128, K)
        assert torch.equal(scale_rows(sf, rb * 128, K), want)
        assert torch.equal(dq[off:off + R * K].view(R, K).float().cpu(), ref.dequantize())
    bias = b[L["b1"]:L["b1"] + 4 * hidden].view(torch.float32)
    assert torch.equal(bias, master[n1:n1 + hidden])
    b2 = b[L["b2"]:L["b2"] + 256].view(torch.float32)
    assert torch.equal(b2[:ncls], master[n1 + hidden + n2:]) and bool((b2[ncls:] == 0).all())
    assert bool((b[L["total"]:] == C_CANARY).all())


# ------------------------------------------------------------------ gemm_mx8: exact fixtures
def to_cuda_nan_padded(m: MX8, extra=32):
    """Copy of m whose pad bytes (K .. pitch) are e4m3 NaN, in a row pitch 32 bytes wider."""
    R, K = m.rows, m.K
    ld = (K + 15) // 16 * 16 + extra
    buf = torch.full((R, ld), 0x7F, dtype=torch.uint8)
    buf[:, :K] = m.q.view(torch.uint8)[:, :K]
    return MX8(buf.cuda().view(torch.float8_e4m3fn), m.sf.cuda(), R, K)


def run_gemm(a, b, bias, alpha, act, dt):
    from bflc_demo_b200.ops.mx8 import gemm_mx8
    M, N = a.rows, b.rows
    ldd = (N + 3) // 4 * 4 + 8
    buf = torch.full((M + 2, ldd + 8), float("nan"), dtype=dt, device="cuda")
    out = buf[1:M + 1, 8:8 + N]
    gemm_mx8(to_cuda_nan_padded(a), to_cuda_nan_padded(b), out=out, out_dtype=dt, alpha=alpha,
             bias=None if bias is None else bias.cuda(), act=act)
    torch.cuda.synchronize()
    keep = torch.ones_like(buf, dtype=torch.bool)
    keep[1:M + 1, 8:8 + N] = False
    assert bool(buf[keep].isnan().all()), "write outside the output"
    return out.cpu()


EXACT = [(1, 1, 16), (64, 3, 32), (127, 5, 48), (128, 62, 100), (129, 63, 128), (300, 64, 784), (64, 65, 4096),
         (129, 127, 100), (128, 128, 48), (300, 129, 784), (4096, 200, 4096), (127, 200, 16), (1, 65, 784),
         (300, 1, 100), (4096, 64, 128), (129, 129, 32), (256, 256, 784), (512, 128, 100)]


@gpu
@pytest.mark.parametrize("M,N,K", EXACT)
def test_gemm_mx8_exact(M, N, K):
    i = EXACT.index((M, N, K))
    for act in (0, 1):
        for with_bias in (False, True):
            dt = torch.float32 if (act + with_bias + i) % 2 == 0 else torch.bfloat16
            a, b, bias, alpha = exact_fixture(M, N, K, seed=i, bias=with_bias, alpha=(0.5, 1.0, 2.0)[i % 3])
            ref = reference_out(a, b, bias, alpha, act)
            got = run_gemm(a, b, bias, alpha, act, dt)
            want = ref.float().to(dt)
            bad = (got != want).nonzero()
            assert bad.numel() == 0, (act, with_bias, dt, bad[:5].tolist())


# ------------------------------------------------------------------ gemm_mx8: rounding-realistic
def gelu64(z):
    return 0.5 * z * (1.0 + torch.special.erf(z / math.sqrt(2.0)))


REAL = [(128, 128, 128), (256, 256, 512), (300, 200, 784), (512, 62, 256), (4096, 1024, 512), (129, 65, 1000)]


@gpu
@pytest.mark.parametrize("M,N,K", REAL)
@pytest.mark.parametrize("act", [0, 1, 2])
def test_gemm_mx8_realistic(M, N, K, act):
    from bflc_demo_b200.ops.mx8 import gemm_mx8, quantize_mx8
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g) * torch.logspace(-2, 1, K)
    b = (torch.randn(N, K, generator=g) * 0.3).bfloat16()
    bias = torch.randn(N, generator=g)
    alpha = 0.7
    qa, qb = quantize_mx8(a.cuda()), quantize_mx8(b.cuda())
    da, db = qa.dequantize().double().cpu(), qb.dequantize().double().cpu()
    assert torch.equal(da, quantize_mx8_reference(a).dequantize().double())
    acc = da @ db.t()
    s_abs = da.abs() @ db.abs().t()
    G = (K + 31) // 32
    z = alpha * acc + bias.double()
    # fp32 sum of each group's 32 exact products, the scaled add per group, the alpha / bias FMA
    err_z = alpha * (32 + G) * U * s_abs + U * (alpha * s_abs + bias.double().abs())
    for dt in (torch.float32, torch.bfloat16):
        out = gemm_mx8(qa, qb, out_dtype=dt, alpha=alpha, bias=bias.cuda(), act=act).float().cpu().double()
        if act == 0:
            ref, err = z, err_z
        elif act == 1:
            ref, err = z.clamp_min(0), err_z
        else:
            # gelu is 1.13-Lipschitz; erff (2 ulp), x * 1/sqrt2, 1 + erf, 0.5 * x, * (...) roundings
            ref = gelu64(z)
            err = 1.13 * err_z + z.abs() * (2 * 2.0 ** -23 + 4 * U) + 4 * U * ref.abs()
        rnd = (2.0 ** -8 if dt == torch.bfloat16 else U) * (ref.abs() + err)
        bound = err + rnd + 2.0 ** -120
        bad = ((out - ref).abs() > bound).nonzero()
        assert bad.numel() == 0, (dt, bad[:5].tolist(), float(((out - ref).abs() / bound).max()))


# ------------------------------------------------------------------ gemm_mx8: scale range
def _range_case(kind):
    K = 64
    a = torch.zeros(1, K)
    b = torch.zeros(4, K)
    if kind == "small_sum":          # ea + eb < 128: both groups' amax near 1e-17
        a[0, :32] = torch.linspace(0.5, 1.0, 32) * 1e-17
        b[:, :32] = torch.linspace(1.0, 0.25, 32) * 1e-17
    elif kind == "zero_partial":     # ea + eb > 381 in a group whose partial is exactly 0
        a[0, 0] = 3e38
        b[:, 1] = 3e38
        a[0, 32:] = 1.0
        b[:, 32:] = 0.5
    else:                            # extreme but in-range pair: ea = 3, eb = 250
        a[0, :32] = 2.0 ** -120
        b[:, :32] = 2.0 ** 120
    return a, b


@gpu
@pytest.mark.parametrize("kind", [
    pytest.param("small_sum", marks=pytest.mark.xfail(strict=True, reason="known: sa * sb underflows")),
    pytest.param("zero_partial", marks=pytest.mark.xfail(strict=True, reason="known: 0 * inf = NaN")),
    "extreme_in_range"])
def test_gemm_mx8_scale_products_out_of_fp32_range(kind):
    """Whenever the exact output is a normal fp32, the kernel must produce it.  The scale fold
    ``part * (sa * sb)`` (wg::mx_accumulate) cannot when the product 2^(ea+eb-254) leaves the
    fp32 range; the first two cases record that defect (DESIGN.md §3.5)."""
    from bflc_demo_b200.ops.mx8 import gemm_mx8, quantize_mx8
    a, b = _range_case(kind)
    qa, qb = quantize_mx8(a.cuda()), quantize_mx8(b.cuda())
    ref = qa.dequantize().double().cpu() @ qb.dequantize().double().cpu().t()
    assert bool((ref.abs() >= 2.0 ** -126).all()) and bool((ref.abs() < 3e38).all())
    out = gemm_mx8(qa, qb, out_dtype=torch.float32).double().cpu()
    assert bool(((out - ref).abs() <= 68 * U * ref.abs()).all()), (out, ref)


# ------------------------------------------------------------------ ops.nn route
@gpu
def test_linear_mx8_route_bit_exact(monkeypatch):
    from bflc_demo_b200.ops import gemm as G
    from bflc_demo_b200.ops import nn as F
    from bflc_demo_b200.ops.mx8 import gemm_mx8, quantize_mx8
    m = Cm()
    log = []
    for name in ("gemm_mx8", "gemm", "quantize_mx8"):
        orig = getattr(m, name)
        monkeypatch.setattr(m, name, (lambda n, o: lambda *a, **k: (log.append(n), o(*a, **k))[1])(name, orig))
    prev = F.set_precision("mx8")
    try:
        torch.manual_seed(3)
        for N, act, want in ((64, G.ACT_NONE, "gemm_mx8"), (64, G.ACT_RELU, "gemm_mx8"),
                             (64, G.ACT_GELU, "gemm"), (62, G.ACT_RELU, "gemm")):
            x = (torch.randn(300, 784, device="cuda") * 0.5).bfloat16()
            w = (torch.randn(N, 784, device="cuda") * 0.05).bfloat16()
            bias = torch.randn(N, device="cuda")
            log.clear()
            y = F.linear(x, w, bias, act=act)
            assert want in log and ({"gemm_mx8", "gemm"} - {want}).isdisjoint(log), (N, act, log)
            if want == "gemm_mx8":
                d = gemm_mx8(quantize_mx8(x), quantize_mx8(w), bias=bias, act=act)
                assert torch.equal(y, d)
    finally:
        F.set_precision(prev)
