"""CPU: the MXFP8 specification (``ops/mx8.py``) that every quantiser and the block-scaled GEMM
are tested against on the GPU.

* The scale-byte rule of the kernels (``epi::mx8_scale_byte``: RN fp32 ``amax * fl(1/448)``,
  flush to zero, biased exponent + "mantissa != 0", clamp to [3, 254]) emulated in numpy, and the
  spec's ``mx8_scale_bytes``, both against the exact rational rule "smallest k with
  448 * 2^k >= amax" on +-256 ulps around every 448 * 2^k, the flush / clamp-to-3 region and
  random amax values.  The fp32 ``ceil(log2(amax / 448))`` formula the spec used before is shown
  to get the boundary groups wrong.
* Flush-to-zero of inputs and of ``x * in_scale``, signed zeros, the e4m3 saturation band.
* The byte-level encoder against its decoder (``MX8.dequantize``).
* The exact GEMM fixtures of ``test_gpu_mx8_conformance.py`` (built here, imported there) are
  exact in fp32 by construction, and a CPU emulation of ``gemm_mx8``'s per-group accumulation
  shows that each plausible kernel mistake changes at least one output element of them.
"""
import math

import numpy as np
import pytest
import torch

from bflc_demo_b200.ops.mx8 import MX8, SF_CHUNK, encode_mx8, mx8_scale_bytes, quantize_mx8_reference

INV448 = np.float32(1.0) / np.float32(448.0)


# ------------------------------------------------------------------ scale-byte rules
def device_scale_byte(amax: np.ndarray) -> np.ndarray:
    """numpy emulation of epi::mx8_scale_byte on fp32 amax (normal or zero: the kernels' inputs
    are flushed before the max)."""
    a = amax.astype(np.float32)
    with np.errstate(over="ignore", under="ignore"):
        p = a * INV448                                         # RN fp32 multiply
    p = np.where(np.abs(p) < np.float32(2.0 ** -126), np.float32(0.0), p)   # .ftz result
    b = p.view(np.uint32)
    e = ((b >> 23) & 0xFF).astype(np.int64) + ((b & 0x7FFFFF) != 0)
    e = np.clip(e, 3, 254)
    return np.where(a > 0, e, 127)


def exact_scale_byte(amax: np.ndarray) -> np.ndarray:
    """Smallest k with 448 * 2^k >= amax, found and verified with exact fp64 ldexp comparisons
    (448 * 2^k and every fp32 amax are exact fp64 values)."""
    a = amax.astype(np.float64)
    _, x = np.frexp(a)
    k = x.astype(np.int64) - 10                                 # 448 * 2^(x-10) < 0.5 * 2^x <= a
    for _ in range(3):
        k = np.where(np.ldexp(448.0, k) < a, k + 1, k)
    pos = a > 0
    assert np.all(np.ldexp(448.0, k[pos]) >= a[pos]) and np.all(np.ldexp(448.0, k[pos] - 1) < a[pos])
    return np.where(pos, np.clip(k + 127, 3, 254), 127)


def old_log2_byte(amax: np.ndarray) -> np.ndarray:
    """The formula the spec used before: fp32 ceil(log2(amax / 448))."""
    t = torch.from_numpy(amax.astype(np.float32))
    return (torch.ceil(torch.log2(t / 448.0)).clamp(-124, 127) + 127).long().numpy()


def boundary_bands(width=256):
    """fp32 values within +-width ulps of 448 * 2^k for every k whose centre is a positive normal
    fp32 (or subnormal, below the flush region of interest), excluding non-normal values."""
    out = []
    for k in range(-134, 120):
        c = np.float32(np.ldexp(448.0, k)) if k > -150 else None
        if c is None or c == 0 or not np.isfinite(c):
            continue
        bits = np.int64(np.array(c, np.float32).view(np.uint32)) + np.arange(-width, width + 1)
        bits = bits[(bits > 0x007FFFFF) & (bits < 0x7F800000)]
        out.append(bits.astype(np.uint32).view(np.float32))
    return np.concatenate(out)


def test_device_rule_and_spec_equal_exact_rule_at_every_binade_boundary():
    a = boundary_bands()
    want = exact_scale_byte(a)
    assert np.array_equal(device_scale_byte(a), want)
    assert np.array_equal(mx8_scale_bytes(torch.from_numpy(a)).long().numpy(), want)


def test_flush_and_clamp_region_and_random_amax():
    rng = np.random.default_rng(0)
    hi = np.array(np.float32(np.ldexp(448.0, -118)), np.float32).view(np.uint32)
    low = rng.integers(0x00800000, int(hi), 200_000, dtype=np.int64).astype(np.uint32).view(np.float32)
    anyf = rng.integers(0x00800000, 0x7F800000, 1_000_000, dtype=np.int64).astype(np.uint32).view(np.float32)
    extremes = np.array([np.finfo(np.float32).tiny, np.finfo(np.float32).max, 448.0, 0.0], np.float32)
    for a in (low, anyf, extremes):
        want = exact_scale_byte(a)
        assert np.array_equal(device_scale_byte(a), want)
        assert np.array_equal(mx8_scale_bytes(torch.from_numpy(a)).long().numpy(), want)
    assert int(mx8_scale_bytes(torch.tensor([np.finfo(np.float32).max])).item()) == 247
    assert int(mx8_scale_bytes(torch.tensor([2.0 ** -126])).item()) == 3


def test_old_log2_formula_fails_just_above_the_boundaries():
    """amax 1, 2 or 3 ulps above 448 * 2^k: fp32 log2 rounds down to exactly k, so the old
    formula picked a scale one binade too small (the group's largest element saturated)."""
    cs = [np.float32(np.ldexp(448.0, k)) for k in range(-120, 110)]
    a = np.array([np.nextafter(np.nextafter(c, np.float32(np.inf)), np.float32(np.inf)) if j == 2 else
                  (np.nextafter(c, np.float32(np.inf)) if j == 1 else
                   np.array(np.array(c, np.float32).view(np.uint32) + 3, np.uint32).view(np.float32))
                  for c in cs for j in (1, 2, 3)], np.float32)
    want = exact_scale_byte(a)
    bad = int((old_log2_byte(a) != want).sum())
    assert bad > len(a) // 2, bad
    assert np.array_equal(mx8_scale_bytes(torch.from_numpy(a)).long().numpy(), want)
    # through the whole reference quantiser: the group's largest element is not saturated
    x = torch.zeros(1, 32)
    x[0, 0] = float(np.nextafter(np.float32(448.0), np.float32(np.inf)))
    m = quantize_mx8_reference(x)
    assert int(m.sf[0].item()) == 128 and float(m.q[0, 0].float()) == 224.0


def test_reference_flushes_inputs_and_products_and_keeps_signs():
    x = torch.zeros(2, 32)
    x[0, :4] = torch.tensor([2.0 ** -130, -(2.0 ** -140), 2.0 ** -126, -0.0])   # subnormals -> +-0
    x[1, :2] = torch.tensor([2.0 ** -100, -(2.0 ** -100)])
    m = quantize_mx8_reference(x)
    codes = m.q.view(torch.uint8)
    assert int(codes[0, 0]) == 0 and int(codes[0, 1]) == 0x80 and int(codes[0, 3]) == 0x80
    assert int(m.sf[0].item()) == 3 and float(m.dequantize()[0, 2]) == 2.0 ** -126
    # x * in_scale = +-2^-130 is flushed although x is normal: an all-zero group, signs kept
    m2 = quantize_mx8_reference(x[1:], in_scale=2.0 ** -30)
    c2 = m2.q.view(torch.uint8)
    assert int(c2[0, 0]) == 0 and int(c2[0, 1]) == 0x80 and int(m2.sf[0].item()) == 127
    # e4m3 saturation band 448..464 and beyond clamps to 448 at the group's scale
    y = torch.zeros(1, 32)
    y[0, :4] = torch.tensor([448.0, 460.0, -463.0, 100.0])
    my = quantize_mx8_reference(y)
    assert int(my.sf[0].item()) == 128                          # 463 > 448: next binade
    assert float(my.q[0, 2].float()) == -224.0                  # 231.5 -> nearest at step 16: 224
    assert float(my.q[0, 1].float()) == 224.0 and float(my.q[0, 0].float()) == 224.0   # 230 / 224


def test_encoder_and_decoder_round_trip():
    g = torch.Generator().manual_seed(1)
    for R, K in [(1, 16), (129, 100), (300, 784)]:
        nz = (K + 31) // 32
        codes = torch.randint(0, 256, (R, (K + 15) // 16 * 16), generator=g, dtype=torch.uint8)
        codes[(codes & 0x7F) == 0x7F] = 0
        e = torch.randint(100, 155, (R, nz), generator=g, dtype=torch.uint8)   # products stay normal fp32
        m = encode_mx8(codes, e, R, K)
        want = codes.view(torch.float8_e4m3fn)[:, :K].double() * torch.exp2(
            e.double() - 127).repeat_interleave(32, 1)[:, :K]
        assert torch.equal(m.dequantize().double(), want)
        kb = (K + 127) // 128
        assert m.sf.numel() == (R + 255) // 256 * 2 * kb * SF_CHUNK
        r, grp = R - 1, nz - 1
        assert int(m.sf[sf_index(r, grp, kb)]) == int(e[r, grp])
    x = torch.randn(129, 100) * torch.logspace(-3, 3, 100)
    ref = quantize_mx8_reference(x)
    again = encode_mx8(ref.q, scale_rows(ref.sf, 129, 100), 129, 100)
    assert torch.equal(again.sf, ref.sf) and torch.equal(again.dequantize(), ref.dequantize())


# ------------------------------------------------------------------ scale-array helpers
def sf_index(row, g, n_kb, transposed=False):
    off = ((row & 127) >> 5) * 32 * 4 + (row & 31) * 4 if transposed else (row & 31) * 16 + ((row & 127) >> 5) * 4
    return ((row >> 7) * n_kb + (g >> 2)) * SF_CHUNK + off + (g & 3)


def scale_rows(sf, rows, K):
    """Chunk array -> [rows, groups] scale bytes (inverse of the encoder's layout)."""
    kb = (K + 127) // 128
    rb = sf.numel() // (kb * SF_CHUNK)
    return sf.view(rb, kb, 32, 4, 4).permute(0, 3, 2, 1, 4).reshape(rb * 128, kb * 4)[:rows]


# ------------------------------------------------------------------ exact GEMM fixtures
def exact_operand(rows, K, seed, ld=None):
    """Small-integer e4m3 codes and scale bytes in [125, 129] drawn independently per (row, group),
    so rows 8, 32, 64 and 128 apart and neighbouring groups carry different bytes at most
    positions (test_fixture_scales_are_not_periodic) and reading any wrong scale shows."""
    g = torch.Generator().manual_seed(seed)
    ld = ld or (K + 15) // 16 * 16
    vals = torch.randint(-3, 4, (rows, K), generator=g).float()
    q = torch.zeros(rows, ld, dtype=torch.float8_e4m3fn)
    q[:, :K] = vals.to(torch.float8_e4m3fn)
    e = torch.randint(125, 130, (rows, (K + 31) // 32), generator=g)
    return encode_mx8(q, e.to(torch.uint8), rows, K)


def exact_fixture(M, N, K, seed=0, bias=True, alpha=0.5):
    a, b = exact_operand(M, K, seed), exact_operand(N, K, seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    bv = (torch.randint(-8, 9, (N,), generator=g) + torch.randint(0, 16, (N,), generator=g) / 16.0).float() \
        if bias else None
    return a, b, bv, alpha


def assert_exact_premise(a, b, bias, alpha):
    """Every partial sum of the GEMM, in any order, and alpha * acc + bias are exact in fp32:
    all terms are multiples of one power of two and the sum of their magnitudes stays below
    2^24 of it."""
    da, db = a.dequantize().double(), b.dequantize().double()
    s_abs = da.abs() @ db.abs().t()
    quantum = 2.0 ** -4 * 2.0 ** math.floor(math.log2(alpha))    # scale bytes >= 125 twice
    if bias is not None:
        assert torch.equal(bias.double() * 16, torch.round(bias.double() * 16))
        quantum = min(quantum, 2.0 ** -4)
        s_abs = alpha * s_abs + bias.double().abs()
    else:
        s_abs = alpha * s_abs
    assert float(s_abs.max()) < 2.0 ** 24 * quantum
    return da, db


def reference_out(a, b, bias, alpha, act):
    da, db = assert_exact_premise(a, b, bias, alpha)
    y = alpha * (da @ db.t())
    if bias is not None:
        y = y + bias.double()
    if act == 1:
        y = y.clamp_min(0.0)
    return y


MUTATIONS = ("transposed_scale_index", "neighbour_k_group", "b_col0_off_by_64", "b_col0_zero",
             "sa1_from_row_r0", "wrong_32_row_subblock", "wrong_128_row_block", "scales_on_wrong_operand",
             "last_k_block_dropped", "bias_shifted")


def remap_rows(rows, mutation):
    """Row whose scale a mutated kernel reads for A row r."""
    if mutation == "sa1_from_row_r0":
        return torch.where(rows % 16 >= 8, rows - 8, rows)
    if mutation == "wrong_32_row_subblock":
        return rows ^ 32
    if mutation == "wrong_128_row_block":
        return rows ^ 128
    return rows


def remap_cols(cols, mutation):
    """Row of B's scale array a mutated kernel reads for output column c (the tile of 64 columns
    starting at n0 reads chunk rows from b_col0 = n0 & 127)."""
    if mutation == "b_col0_off_by_64":
        return (cols & ~127) | ((cols & 127) ^ 64)
    if mutation == "b_col0_zero":
        return torch.where((cols & 127) >= 64, cols - 64, cols)
    return cols


def emulate_gemm_mx8(a, b, bias, alpha, act, mutation=None):
    """fp64 emulation of gemm_mx8_kernel's per-group accumulation, reading the scales out of the
    chunk arrays the way the kernel does; `mutation` injects one kernel mistake."""
    M, N, K = a.rows, b.rows, a.K
    kb = (K + 127) // 128
    G = (K + 31) // 32
    qa = a.q[:, :K].double()
    qb = b.q[:, :K].double()
    rows = torch.arange(M)
    cols = torch.arange(N)
    out = torch.zeros(M, N, dtype=torch.float64)
    for g in range(G):
        if mutation == "last_k_block_dropped" and g >= (kb - 1) * 4:
            break
        gs = g ^ 1 if mutation == "neighbour_k_group" else g
        ra, cb = remap_rows(rows, mutation), remap_cols(cols, mutation)
        tr = mutation == "transposed_scale_index"
        if mutation == "scales_on_wrong_operand":
            sa_src, sb_src, ra, cb = b.sf, a.sf, ra % N, cb % M
        else:
            sa_src, sb_src = a.sf, b.sf
        ia = torch.tensor([sf_index(int(r), gs, kb, tr) for r in ra])
        ib = torch.tensor([sf_index(int(c), gs, kb, tr) for c in cb])
        ea = sa_src[ia].double() - 127
        eb = sb_src[ib].double() - 127
        part = qa[:, g * 32:(g + 1) * 32] @ qb[:, g * 32:(g + 1) * 32].t()
        out += part * torch.exp2(ea).view(-1, 1) * torch.exp2(eb).view(1, -1)
    out = alpha * out
    if bias is not None:
        bb = bias.double()
        if mutation == "bias_shifted":
            bb = torch.cat([bb[1:], bb.new_zeros(1)])
        out = out + bb
    return out.clamp_min(0.0) if act == 1 else out


def test_emulation_matches_fp64_product_on_exact_fixtures():
    for M, N, K in [(129, 65, 100), (300, 200, 784), (1, 3, 16)]:
        a, b, bias, alpha = exact_fixture(M, N, K)
        ref = reference_out(a, b, bias, alpha, 1)
        assert torch.equal(emulate_gemm_mx8(a, b, bias, alpha, 1), ref)
        assert torch.equal(ref.float().double(), ref)              # exact in fp32


def test_fixture_scales_are_not_periodic():
    for rows, K in [(4096, 4096), (300, 784)]:
        e = scale_rows(exact_operand(rows, K, 0).sf, rows, K).long()
        for d in (8, 32, 64, 128):
            same = float((e[d:] == e[:-d]).float().mean())
            assert same < 0.3, (rows, K, d, same)
        assert float((e[:, 1:] == e[:, :-1]).float().mean()) < 0.3


MUTATION_SHAPES = [(256, 256, 784), (256, 128, 100), (512, 256, 4096)]


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_exact_fixtures_detect_each_kernel_mistake(mutation):
    """The GPU suite compares bit for bit, so any changed element fails it.  Every shape here
    keeps each remapped scale index on a real row (no padding byte 0x7F stands in for a real one),
    and each shape on its own must expose the mistake."""
    for M, N, K in MUTATION_SHAPES:
        assert int(remap_rows(torch.arange(M), mutation).max()) < M
        assert int(remap_cols(torch.arange(N), mutation).max()) < N
        a, b, bias, alpha = exact_fixture(M, N, K)
        ref = reference_out(a, b, bias, alpha, 0)
        got = emulate_gemm_mx8(a, b, bias, alpha, 0, mutation)
        assert not torch.equal(got.float(), ref.float()), (mutation, M, N, K)
