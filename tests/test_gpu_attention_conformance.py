"""Conformance of the fused attention kernels (``csrc/kernels/attn_sm100.cu``) against a plain
float64 reference of masked, optionally dropped-out softmax attention, element by element.

Reference (``ref_fwd`` / ``ref_bwd``, fp64 on any device, from the bf16 inputs as stored).  Heads are
[G = B*H, S, 64]; ``kmask`` [G, S] marks the valid keys of each head.
* Padded mode: sequence b attends to keys j < clamp(lengths[b], 0, S); query rows past the length
  are still computed; a length <= 0 gives exactly zero O, lse, dQ, dK and dV; masked keys get
  exactly zero dK and dV.
* Packed mode: sequence b is rows [cu[b], cu[b+1]) and attends within itself.  The reference runs on
  the sequences gathered into [B, S_pad] with the rows past the length masked out; rows outside
  every sequence are never written; lse / delta are [B*H, S_pad], indexed by the in-sequence row.
* Dropout: the keep mask Z is ``test_dropout_host.attention_keep_ref`` (numpy Philox, independent of
  the kernels); O = (P Z / (1-p)) V and dS = P (Z dP / (1-p) - delta) scale, with 1 / (1-p) the fp32
  value the launcher computes.
``test_reference_matches_autograd`` checks the reference against fp64 scaled_dot_product_attention
and autograd.

Per stage, from the kernel's own intermediates: the forward is checked on O and lse; the backward on
delta, dQ, dK and dV against fp64 computed from the kernel's bf16 O and fp32 lse (P = exp(scale s -
lse_kernel), delta = rowsum(dO O_kernel)), so a forward error is never charged to the backward.

Bound model (``fwd_bounds`` / ``bwd_bounds``), built from fp64 products of absolute values, with no
fitted constant.  u = 2^-24 is one rounding to nearest, one fp32 ulp 2^-23 is used where the
hardware may truncate (tensor-core sums), gamma_n = n 2^-23 / (1 - n 2^-23).  The build uses
--use_fast_math, so exp2f is ex2.approx.ftz (2 ulp, results below 2^-126 flushed to 0), 1.f / x is
an approximate reciprocal (2 ulp), __logf is lg2.approx based (2^-21.41 absolute on [0.5, 2], 3 ulp
elsewhere) -- the CUDA C++ Programming Guide's bounds.  Rounding points: the fp32 sums of q.k, dO.V
and delta over 64 terms (gamma_64 |q||k|^T ...); the exponent arguments (one rounding per operation
on |scale s|, |lse|); P and dS rounded to bf16 before each wgmma (2^-8 relative); l summed in fp32
from the unrounded p; fp32 accumulation over up to 512 keys or queries; the per-block alpha and
1 / l multiplies; the bf16 output (half an ulp, 2^-8 of |out|).

Fixtures (``fixture``):
* E1 hard argmax -- queries are 16 x a +-1 Hadamard row of one target key, other valid keys are 0, so
  every non-target score sits >= 128 below the max in the ex2 argument and flushes to exactly 0: P
  is one-hot, O must equal V[target] bit for bit, dV the exact sum of the dO rows choosing each key,
  dQ = dK = 0.  Variants: every query targets the first key, the last valid key, spread targets,
  masked keys scoring above every valid key (padded), and the next packed sequence's first rows
  scoring above every key of the previous one.
* E2 ties -- groups of 2 or 4 keys share a code, and a shared coordinate (dim 63) shifts each row's
  max score to exactly 0, so P = 1/2 or 1/4 exactly and every result is a small dyadic number.
* R realistic -- random normal q, k, v at scale 0.7 and 2.0 (peaked rows).
* A adversarial online softmax -- the row max rises in every key block (alpha < 1 every step), the
  max sits in block 0 and later blocks are >= 120 below it in scale*s (exact underflow), and
  |scale s| ~ 90 (overflow without the max subtraction).
E1 / E2 premises are asserted in fp64 (``exact_expectation``; CPU guard tests run them on every
exact GPU case).

Case matrix (test ids: route-S-lengths-H-ld-p-fixture):
* whole: the one-CTA-per-head ``attn_fwd_kernel`` / ``attn_bwd_kernel`` (lengths None, S = 128, no
  dropout), B in {1, 3} x H in {1, 4, 12}, plus every fixture and a wide row pitch.
* tiled (``attn_{fwd,dq,dkv}_var_kernel<false, false>``): S in {64, 128, ..., 512}, each with the
  lengths {-3, 0, 1, 63, 64, 65, 127, 128, 129, S-1, S, S+7} (so S = 64 mod 128 runs a query block
  with one live warpgroup), lengths None for S != 128, S = 128 with all lengths S, every fixture at
  S = 448 / 320, a wide pitch.
* packed (``<true, false>``): lengths {1, 63, 64, 65, 128, 129, 511, 512} in mixed orders, zero-length
  sequences in the middle and at the end, offsets that are not multiples of 64, T not a multiple of
  64, trailing rows past cu[B], max_seqlen equal to and above the true max and not a multiple of
  64, a wide pitch.
* dropout (``<false, true>``, ``<true, true>``): p in {0.1, 0.5} x padded / packed x S in {64, 192,
  512}, and unmasked S = 128 (which runs the tiled kernels), wide pitches.
Row pitch: ld = H*64 + 72 means q ... dv are column slices of wider buffers.  Every output buffer
(column gaps, unwritten packed rows, lse / delta tails) starts as a NaN canary, and every canary
outside the written region must survive.  Route: the whole-route backward never writes delta, so
its NaN canary survives everywhere; the tiled routes write delta for every row, checked against
fp64.  ``test_public_ops_match_binding`` covers the routing in ``ops/nn.py``.

``test_bounds_have_teeth`` (CPU) shows the bounds are tighter than the effect of including key
len_b, dropping the last key block, skipping the alpha rescale, a scale off by 2^-7, two heads
swapped, a forgotten 1 / (1-p) and delta = 0, on at least one element of every affected output.
"""
import math
import zlib
from typing import NamedTuple, Optional

import numpy as np
import pytest
import torch

from test_dropout_host import attention_keep_ref

gpu = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
D = 64
SCALE = 0.125                          # 1 / sqrt(64), what ops.nn passes
U = 2.0 ** -24                         # one fp32 rounding to nearest
ULP = 2.0 ** -23                       # one fp32 ulp (covers truncating tensor-core sums)
EX2 = 2 * ULP                          # ex2.approx.ftz.f32: 2 ulp
RCP = 2 * ULP                          # 1.f / x under fast math: 2 ulp
LOGF_ABS, LOGF_REL = 2.0 ** -21.41, 3 * ULP   # __logf: absolute on [0.5, 2], ulp elsewhere
BF_U = 2.0 ** -8                       # bf16 rounding to nearest: half an ulp, relative
FTZ = 2.0 ** -126                      # ex2.approx.ftz flushes results below this to 0
LOG2E = 1.4426950408889634
SEED, STEP, ADD, SITE = 0x0123_4567_89AB_CDEF, 9, 2, 5
CANARY = float("nan")


def gamma(n):
    return n * ULP / (1 - n * ULP)


def dscale_of(p):
    """1 / (1 - p) as the launcher computes it: fp32 division of fp32 values."""
    one = torch.tensor(1.0, dtype=F32)
    return float(one / (one - torch.tensor(p, dtype=F32)))


def bf(t):
    return t.to(BF16).to(F64)


# ----------------------------------------------------------------------- float64 reference
def ref_fwd(q, k, v, kmask, scale, zs=None):
    """q, k, v [G, S, 64] fp64, kmask [G, S] (valid keys), zs [G, S, S] = Z / (1-p) or None.
    -> s, P (softmax over the valid keys), O, lse; a head with no valid key gives P = O = lse = 0."""
    s = q @ k.mT
    x = (scale * s).masked_fill(~kmask[:, None, :], -math.inf)
    has = kmask.any(-1)[:, None]
    lse = torch.where(has, torch.logsumexp(x, -1), 0.0)
    P = torch.exp(x - lse[..., None])
    W = P if zs is None else P * zs
    return {"s": s, "P": P, "o": W @ v, "lse": lse}


def ref_bwd(q, k, v, do, o, lse, kmask, scale, zs=None, qmask=None):
    """Backward from given O and lse (the kernel's): P = exp(scale s - lse) on the valid keys (and
    query rows, ``qmask``), delta = rowsum(dO O), dS = P (Z dP / (1-p) - delta) scale."""
    s = q @ k.mT
    valid = kmask[:, None, :] if qmask is None else kmask[:, None, :] & qmask[:, :, None]
    P = torch.exp((scale * s - lse[..., None]).masked_fill(~valid, -math.inf))
    delta = (do * o).sum(-1)
    dP = do @ v.mT
    Gd = dP if zs is None else zs * dP
    dS = P * (Gd - delta[..., None]) * scale
    W = P if zs is None else P * zs
    return {"s": s, "P": P, "dP": dP, "G": Gd, "dS": dS, "delta": delta,
            "dq": dS @ k, "dk": dS.mT @ q, "dv": W.mT @ do}


# ------------------------------------------------------------------- derived rounding bounds
def fwd_bounds(q, k, v, kmask, scale, ref, zs=None, dscale=1.0):
    """Elementwise bounds on |O_kernel - O| (before the bf16 output rounding) and |lse_kernel - lse|.

    p_ij = ex2((s_ij - m) sc): the score error gamma_64 |q||k|^T, on s_ij and on the row max m, and
    one rounding each for the subtraction, the multiply and sc = scale log2e itself (4 u |x|) move
    the exponent by dx, so p has relative error 2^dx (1 + 2 ulp) - 1 =: rp.  l sums the unrounded p
    in fp32 (gamma over 64 per block) and is multiplied by alpha once per key block; O sums bf16(p) V
    (2^-8, gamma over the keys) and is multiplied by the same alphas, so alpha's own error cancels in
    O = o / l but not in lse.  Then 1 / l (2 ulp), the product (u), and 1 / (1-p) (u) with dropout.
    A p below 2^-126 may flush to 0: at most 2^-126 of a sum l >= 1 per key.
    lse = m scale + __logf(l): scale times the score error, -log(1 - l's relative error, alpha's
    included), __logf's error, and the roundings of m scale and of the sum."""
    km = kmask[:, None, :]
    has = kmask.any(-1)[:, None, None]
    s, P = ref["s"], ref["P"]
    es = gamma(D) * (q.abs() @ k.abs().mT)
    m = torch.where(has, s.masked_fill(~km, -math.inf).amax(-1, keepdim=True), 0.0)
    esm = es.masked_fill(~km, 0).amax(-1, keepdim=True)
    sc = scale * LOG2E
    x = ((s - m) * sc).masked_fill(~km, 0).abs()
    dx = sc * (es + esm) * (1 + U) + 4 * U * x
    rp = (torch.exp2(dx) * (1 + EX2) - 1).masked_fill(~km, 0)
    n = kmask.sum(-1).to(F64)[:, None, None]
    nkb = torch.ceil(n / 64)
    g = 1 + gamma(64 * nkb)
    chain = (1 + ULP) ** nkb
    rpm = rp.amax(-1, keepdim=True)
    rl = (1 + rpm) * g * chain - 1
    rest = (1 + BF_U) * g * chain * (1 + RCP) * (1 + U) * (1 + (U if zs is not None else 0))
    rw = (1 + rp) * rest / (1 - rl) - 1
    W = P if zs is None else P * zs
    ob = (W * rw) @ v.abs() + FTZ * dscale * (km.to(F64) @ v.abs())
    ra = (torch.exp2(4 * U * x.amax(-1, keepdim=True)) * (1 + EX2)) ** nkb
    el = (1 + rpm) * g * chain * ra - 1 + n * FTZ
    lse = ref["lse"][..., None]
    lb = (scale * esm * (1 + U) - torch.log1p(-el) + LOGF_ABS
          + LOGF_REL * (torch.log(n.clamp(min=1)) + el) + 2 * U * (scale * m.abs() + lse.abs() + 1))
    return {"o": ob * has, "lse": (lb * has)[..., 0]}


def bwd_bounds(q, k, v, do, o, lse, kmask, scale, ref, zs=None, dscale=1.0, qmask=None, nq_acc=None):
    """Elementwise bounds on |delta|, |dQ|, |dK|, |dV| errors against ``ref_bwd`` (same O, lse).

    p = ex2(s sc - lse log2e): the score error and one rounding each on |s sc| (product, sc) and
    |lse log2e| (product, log2e) and the difference give rp as in ``fwd_bounds``.  dP and delta
    are fp32 sums of 64 exact bf16 products (gamma_64); with dropout dP / (1-p) rounds once; the
    subtraction and the product with p round once each; dS rounds to bf16 (2^-8) before the dQ
    (gamma over the keys) and dK (gamma over the queries) wgmma.  dV sums bf16(p Z) dO over the
    queries and multiplies by 1 / (1-p) (u) at the end.  Flushed p: 2^-126 each."""
    valid = kmask[:, None, :] if qmask is None else kmask[:, None, :] & qmask[:, :, None]
    vf = valid.to(F64)
    n = kmask.sum(-1).to(F64)[:, None, None]
    nk_acc = 64 * torch.ceil(n / 64)
    if nq_acc is None:
        nq_acc = float(q.shape[1])
    sc = scale * LOG2E
    es = gamma(D) * (q.abs() @ k.abs().mT)
    dx = sc * es * (1 + U) + 3 * U * (ref["s"].abs() * sc + lse.abs()[..., None] * LOG2E)
    rp = (torch.exp2(dx) * (1 + EX2) - 1) * vf
    P = ref["P"]
    edp = gamma(D) * (do.abs() @ v.abs().mT)
    ed = gamma(D) * (do.abs() * o.abs()).sum(-1)
    z = 1.0 if zs is None else zs
    eG = z * edp + (U * z * ref["dP"].abs() if zs is not None else 0)
    A = (ref["G"] - ref["delta"][..., None]).abs()
    eA = eG + ed[..., None] + U * (A + eG + ed[..., None])
    e_pre = scale * (P * rp * A + P * (1 + rp) * eA + U * P * (1 + rp) * (A + eA) + FTZ * (A + eA) * vf)
    edS = e_pre + BF_U * (ref["dS"].abs() + e_pre)
    adS = ref["dS"].abs() + edS
    dq = edS @ k.abs() + gamma(nk_acc) * (adS @ k.abs())
    dk = edS.mT @ q.abs() + gamma(nq_acc) * (adS.mT @ q.abs())
    Z = vf if zs is None else (zs > 0).to(F64) * vf
    Wz = P * Z
    ewb = Wz * rp + FTZ * Z
    ewb = ewb + BF_U * (Wz + ewb)
    aW = (Wz + ewb).mT @ do.abs()
    pre = ewb.mT @ do.abs() + gamma(nq_acc) * aW
    dv = pre if zs is None else dscale * pre * (1 + U) + U * dscale * aW
    return {"delta": ed, "dq": dq, "dk": dk, "dv": dv}


def violations(out, ref, bound, bf16_out=True):
    """Elements with |out - ref| > bound (+ half a bf16 ulp of the result for bf16 outputs)."""
    tol = bound + (BF_U * (ref.abs() + bound) if bf16_out else 0) + FTZ
    return ~torch.isfinite(out) | ((out - ref).abs() > tol)


def _report(bad, what):
    nbad = int(bad.sum())
    if nbad:
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: {nbad} of {bad.numel()} elements wrong, first at {idx}")


# ------------------------------------------------------------------------------- fixtures
def hadamard(n):
    h = torch.ones(1, 1, dtype=F64)
    while h.shape[0] < n:
        h = torch.cat([torch.cat([h, h], 1), torch.cat([h, -h], 1)], 0)
    return h


def sparse_ints(g, *shape):
    """Values in {-1, 0, 1}, three quarters zeros: small exact sums."""
    r = torch.randint(0, 8, shape, generator=g)
    return ((r == 0).to(F64) - (r == 1).to(F64))


def _e1_head(g, q, k, n, S, variant, half, first_rows):
    """One (sequence, head) of E1 into q, k [S, 64].  Targets get distinct Hadamard codes from the
    sequence's half of the 64 rows (alternating by sequence), keys of first_rows carry twice a code
    of the previous packed sequence (they are targets here too)."""
    codes = hadamard(64)
    pool = list(range(32 * half, 32 * half + 32))
    if n <= 0:
        return
    r0 = len(first_rows)
    if variant == "first":
        own = [0] if r0 == 0 else []
    elif variant == "last":
        own = [n - 1] if n - 1 >= r0 else []
    else:
        cand = list(range(r0, n))
        pick = torch.randperm(len(cand), generator=g)[:28].tolist()
        own = sorted({cand[i] for i in pick} | ({r0, n - 1} if r0 < n else set()))
    targets = []
    for j, c in first_rows:
        k[j] = 2 * codes[c]
        targets.append(c)
    for t, j in enumerate(own):
        k[j] = codes[pool[t]]
        targets.append(pool[t])
    for i in range(S):
        q[i] = 16 * codes[targets[i % len(targets)]]
    if variant == "masked_high":                    # masked keys score twice the max
        for r, j in enumerate(range(n, min(S, n + 8))):
            k[j] = 2 * codes[targets[r % len(targets)]]


def _e2_head(g, q, k, n, S):
    """One (sequence, head) of E2: groups of 2 / 4 valid keys share code h_a (dims 0..31); every
    valid key has dim 63 = 1, queries 32 h_a and dim 63 = -1024, so each row's max score is exactly
    0 and every other valid key scores -1024.  Each key has one entry in dims 32..62 (zero in the
    queries), so tied keys differ and dQ is not trivial.
    Masked keys carry a code with dim 63 = 0: they would score +1024."""
    codes = hadamard(32)
    if n <= 0:
        return
    k[torch.arange(S), 32 + torch.randint(0, 31, (S,), generator=g)] = sparse_ints(g, S)   # one of dims 32..62
    k[:n, 63] = 1
    perm = torch.randperm(n, generator=g).tolist()
    groups, pos = [], 0
    while len(groups) < 24:
        t = (2, 4)[len(groups) % 2]
        if n - pos < t:                             # a shorter group would not be a tie of 2 / 4
            t = 2 if n - pos >= 2 else (1 if not groups else 0)
        if t == 0:
            break
        groups.append(perm[pos:pos + t])
        pos += t
    gc = torch.randperm(32, generator=g)[:len(groups)].tolist()
    for grp, c in zip(groups, gc):
        for j in grp:
            k[j, :32] = codes[c]
    for i in range(S):
        c = gc[int(torch.randint(0, len(groups), (1,), generator=g))]
        q[i, :32] = 32 * codes[c]
        q[i, 63] = -1024
    for j in range(n, S):
        k[j, :32] = codes[gc[j % len(gc)]]


def fixture(name, B, S, H, n, packed=False, seed=0):
    """q, k, v, dO as fp64 [B, S, H, 64], exactly bf16; n[b] the valid length of sequence b."""
    g = torch.Generator().manual_seed(seed)
    shape = (B, S, H, D)
    if name.startswith("E"):
        q, k = torch.zeros(shape, dtype=F64), torch.zeros(shape, dtype=F64)
        v = torch.randint(-8, 9, shape, generator=g).to(F64) if name != "E2" else sparse_ints(g, *shape)
        do = sparse_ints(g, *shape)
        prev = None
        for b in range(B):
            for h in range(H):
                if name == "E2":
                    _e2_head(g, q[b, :, h], k[b, :, h], n[b], S)
                    continue
                variant = name.split("-")[1]
                first = []
                if variant == "next_high" and prev is not None:
                    first = [(j, 32 * (prev % 2) + j) for j in range(min(4, n[b]))]
                _e1_head(g, q[b, :, h], k[b, :, h], n[b], S, variant, b % 2, first)
            if n[b] > 0:
                prev = b
        return q, k, v, do
    sd = {"R0.7": 0.7, "R2": 2.0}.get(name, 0.7)
    q, k, v = (bf(torch.randn(shape, generator=g, dtype=F64) * sd) for _ in range(3))
    do = bf(torch.randn(shape, generator=g, dtype=F64))
    blk = (torch.arange(S) // 64).to(F64)[None, :, None]
    if name == "A-rise":                            # +2 in scale*s per key block
        q[..., 63], k[..., 63] = 8.0, 2.0 * blk
    elif name == "A-under":                         # blocks >= 1 sit 128 below block 0 in scale*s
        q[..., 63], k[..., 63] = 16.0, -64.0 * (blk > 0)
    elif name == "A-big":                           # scale*s ~ 90
        q[..., 63], k[..., 63] = 32.0, 22.5
    return q, k, v, do


def heads(x):
    B, S, H, _ = x.shape
    return x.permute(0, 2, 1, 3).reshape(B * H, S, D)


def masks(n, S, H, packed):
    """kmask [G, S] (keys j < n_b) and qmask [G, S] (packed: rows i < n_b; padded: all)."""
    nn_ = torch.tensor(n).repeat_interleave(H)[:, None]
    j = torch.arange(S)[None, :]
    kmask = j < nn_
    return kmask, (kmask.clone() if packed else torch.ones_like(kmask))


def ideal_p(s, kmask, scale):
    """P of an exact fixture: 1 / t on the t keys attaining the row max, 0 elsewhere, after asserting
    that every other valid key's ex2 argument is <= -128 (ex2.approx.ftz returns exactly 0)."""
    km = kmask[:, None, :]
    has = kmask.any(-1)[:, None, None]
    m = torch.where(has, s.masked_fill(~km, -math.inf).amax(-1, keepdim=True), 0.0)
    top = (s == m) & km
    gap = ((s - m) * scale * LOG2E).masked_fill(top | ~km, -math.inf)
    assert float(gap.amax()) <= -128.0, "runner-up too close to the max"
    t = top.sum(-1, keepdim=True)
    assert bool(((t == 0) | (t == 1) | (t == 2) | (t == 4)).all())
    return top.to(F64) / t.clamp(min=1)


def _dyadic_exp(x):
    for e in range(0, 40):
        if bool((x * 2.0 ** e == torch.round(x * 2.0 ** e)).all()):
            return e
    raise AssertionError("not dyadic")


def assert_sum_exact(A, Bm, what):
    """Every fp32 partial sum of A @ Bm (any order) is exact: all terms on a 2^-e grid and
    sum |a||b| < 2^24 grid steps."""
    e = _dyadic_exp(A) + _dyadic_exp(Bm)
    assert float((A.abs() @ Bm.abs()).amax()) * 2.0 ** e < 2.0 ** 24, what


def exact_expectation(q, k, v, do, kmask, qmask, scale):
    """E1 / E2 premises and the exact results (P ideal, O, delta, dQ, dK, dV), heads form."""
    for t in (q, k, v, do):
        assert torch.equal(bf(t), t)
    s = q @ k.mT
    assert_sum_exact(q, k.mT, "scores")
    P = ideal_p(s, kmask, scale) * qmask[:, :, None]
    o = P @ v
    assert_sum_exact(P, v, "P V")
    assert torch.equal(bf(o), o), "O not bf16"
    do = do * qmask[..., None]
    delta = (do * o).sum(-1)
    assert_sum_exact((do * o), torch.ones(D, 1, dtype=F64, device=q.device), "delta")
    assert_sum_exact(do, v.mT, "dP")
    dS = P * (do @ v.mT - delta[..., None]) * scale
    assert torch.equal(bf(dS), dS), "dS not bf16"      # so p's ex2 / __logf error cannot move it
    out = {"P": P, "o": o, "delta": delta, "dq": dS @ k, "dk": dS.mT @ q, "dv": P.mT @ do}
    for name, (a, b) in {"dq": (dS, k), "dk": (dS.mT, q), "dv": (P.mT, do)}.items():
        assert_sum_exact(a, b, name)
        assert torch.equal(bf(out[name]), out[name]), f"{name} not bf16"
    return out


# --------------------------------------------------------------------------------- cases
class Case(NamedTuple):
    route: str                      # whole | tiled | packed
    S: int                          # padded S; packed: max_seqlen
    lens: Optional[tuple]           # padded: lengths (None: no mask); packed: sequence lengths
    H: int
    fx: str = "R0.7"
    B: int = 0                      # padded, lens None
    ld: int = 0                     # extra row pitch beyond H*64
    p: float = 0.0
    trail: int = 0                  # packed: rows past cu[B]

    @property
    def nseq(self):
        return self.B if self.lens is None else len(self.lens)

    @property
    def S_pad(self):
        return (self.S + 63) // 64 * 64

    def valid(self):
        if self.route == "packed":
            return [min(x, self.S_pad) for x in self.lens]
        if self.lens is None:
            return [self.S] * self.nseq
        return [min(max(x, 0), self.S) for x in self.lens]

    def id(self):
        ln = f"none.B{self.B}" if self.lens is None else ("edges" if self.lens == edge_lens(self.S) else
                                                ".".join(str(x) for x in self.lens))
        tr = f"+{self.trail}" if self.trail else ""
        return f"{self.route}-S{self.S}-{ln}{tr}-H{self.H}-ld{self.H * D + self.ld}-p{self.p}-{self.fx}"


def edge_lens(S):
    return (-3, 0, 1, 63, 64, 65, 127, 128, 129, S - 1, S, S + 7)


SS = (64, 128, 192, 256, 320, 384, 448, 512)
PK1 = (1, 63, 64, 65, 128, 129, 511, 512)
PK2 = (512, 0, 129, 65, 0, 1, 64, 63, 128, 511, 0)
PK3 = (65, 129, 0, 63, 100)
FIXTURES = ("R2", "A-rise", "A-under", "A-big", "E1-first", "E1-last", "E1-spread", "E1-masked_high", "E2")

CASES = (
    [Case("whole", 128, None, h, B=b) for b in (1, 3) for h in (1, 4, 12)]
    + [Case("whole", 128, None, 4, fx, B=3) for fx in FIXTURES if fx != "E1-masked_high"]
    + [Case("whole", 128, None, 4, B=2, ld=72)]
    + [Case("tiled", S, edge_lens(S), 2) for S in SS]
    + [Case("tiled", S, None, 2, B=2) for S in SS if S != 128]
    + [Case("tiled", 128, (128, 128, 128), 2)]
    + [Case("tiled", 448, edge_lens(448), 2, fx) for fx in FIXTURES]
    + [Case("tiled", 192, edge_lens(192), 2, fx) for fx in ("E1-first", "E1-last", "E2")]
    + [Case("tiled", 320, edge_lens(320), 2, ld=72), Case("tiled", 320, edge_lens(320), 3, "E1-spread", ld=72)]
    + [Case("packed", 512, PK1, 2), Case("packed", 512, PK2, 2, trail=37), Case("packed", 129, PK3, 3),
       Case("packed", 200, PK3, 2, trail=5), Case("packed", 512, PK2, 2, "R2"),
       Case("packed", 512, PK1, 2, "A-rise"), Case("packed", 512, PK2, 2, "A-under", trail=11),
       Case("packed", 512, PK1, 2, "E1-next_high"), Case("packed", 512, PK2, 2, "E1-next_high", trail=64),
       Case("packed", 129, PK3, 2, "E1-spread"), Case("packed", 512, PK1, 2, "E2"),
       Case("packed", 512, PK2, 2, ld=72, trail=3), Case("packed", 200, PK3, 2, "E1-next_high", ld=72)]
    + [Case("tiled", S, edge_lens(S), 2, p=p) for p in (0.1, 0.5) for S in (64, 192, 512)]
    + [Case("packed", S, lens, 2, p=p, trail=7) for p in (0.1, 0.5)
       for S, lens in ((64, (64, 1, 0, 63, 17)), (192, (192, 65, 0, 129, 1)), (512, PK2))]
    + [Case("tiled", 128, None, 2, B=3, p=0.1), Case("tiled", 192, edge_lens(192), 2, p=0.5, ld=72),
       Case("packed", 192, (192, 65, 0, 129, 1), 2, p=0.1, ld=72)]
)
EXACT_CASES = [c for c in CASES if c.fx.startswith("E")]


def case_data(c, dev="cpu"):
    """Fixture tensors [B, S', H, 64] (S' = S_pad for packed) and the masks, on ``dev``."""
    S = c.S_pad if c.route == "packed" else c.S
    n = c.valid()
    q, k, v, do = fixture(c.fx, c.nseq, S, c.H, n, c.route == "packed", seed=zlib.crc32(c.id().encode()))
    kmask, qmask = masks(n, S, c.H, c.route == "packed")
    to = lambda t: t.to(dev)  # noqa: E731
    return [to(t) for t in (q, k, v, do)], to(kmask), to(qmask), n, S


# ------------------------------------------------------------------------- CPU: reference
def test_reference_matches_autograd():
    """ref_fwd / ref_bwd against fp64 scaled_dot_product_attention + autograd with a boolean key
    mask, and against autograd of the explicit dropout form; an empty head gives zeros."""
    g = torch.Generator().manual_seed(3)
    G, S = 4, 192
    q, k, v, do = (torch.randn(G, S, D, generator=g, dtype=F64) for _ in range(4))
    lens = torch.tensor([192, 65, 1, 0])
    kmask = torch.arange(S)[None, :] < lens[:, None]
    keep = torch.rand(G, S, S, generator=g) > 0.3
    for zs in (None, keep.to(F64) / 0.7):
        qa, ka, va = (t.clone().requires_grad_(True) for t in (q, k, v))
        if zs is None:
            o = torch.nn.functional.scaled_dot_product_attention(qa[:3], ka[:3], va[:3], attn_mask=kmask[:3, None, :],
                                                                  scale=SCALE)
        else:
            x = (SCALE * qa[:3] @ ka[:3].mT).masked_fill(~kmask[:3, None, :], -math.inf)
            o = (torch.softmax(x, -1) * zs[:3]) @ va[:3]
        o.backward(do[:3])
        r = ref_fwd(q, k, v, kmask, SCALE, zs)
        torch.testing.assert_close(r["o"][:3], o.detach(), rtol=1e-12, atol=1e-12)
        b = ref_bwd(q, k, v, do, r["o"], r["lse"], kmask, SCALE, zs)
        for name, t in (("dq", qa), ("dk", ka), ("dv", va)):
            torch.testing.assert_close(b[name][:3], t.grad[:3], rtol=1e-10, atol=1e-12)
        x = (SCALE * q[:3] @ k[:3].mT).masked_fill(~kmask[:3, None, :], -math.inf)
        torch.testing.assert_close(r["lse"][:3], torch.logsumexp(x, -1), rtol=1e-14, atol=0)
        for t in (r["o"][3], r["lse"][3], b["dq"][3], b["dk"][3], b["dv"][3]):
            assert not bool(t.any())
        assert not bool(b["dk"][1, 65:].any()) and not bool(b["dv"][1, 65:].any())


@pytest.mark.parametrize("case", EXACT_CASES, ids=lambda c: c.id())
def test_exact_fixture_premises(case):
    """Every premise of an E1 / E2 GPU case, in fp64 on the CPU (see ``exact_expectation``)."""
    (q, k, v, do), kmask, qmask, n, S = case_data(case)
    e = exact_expectation(heads(q), heads(k), heads(v), heads(do), kmask, qmask, SCALE)
    assert bool(e["o"].any()) and bool(e["dv"].any())
    if case.fx == "E2":
        assert bool(e["dk"].any()) and bool(e["dq"].any())
        assert bool((e["P"] == 0.5).any()) and bool((e["P"] == 0.25).any())   # ties of 2 and of 4


# ------------------------------------------------------------------ CPU: the bounds have teeth
def _skip_alpha(q, k, v, kmask, scale):
    """Online softmax without rescaling earlier key blocks when the running max rises."""
    s = q @ k.mT
    G, S, _ = s.shape
    m = torch.full((G, S, 1), -math.inf, dtype=F64)
    o = torch.zeros(G, S, D, dtype=F64)
    l = torch.zeros(G, S, 1, dtype=F64)
    for j0 in range(0, S, 64):
        blk = s[..., j0:j0 + 64].masked_fill(~kmask[:, None, j0:j0 + 64], -math.inf)
        m = torch.maximum(m, blk.amax(-1, keepdim=True))
        p = torch.exp(scale * (blk - m)).nan_to_num(0.0)
        o = o + p @ v[:, j0:j0 + 64]
        l = l + p.sum(-1, keepdim=True)
    return {"o": o / l.clamp(min=1e-300), "lse": (scale * m + torch.log(l))[..., 0]}


def _swap(t, H):
    t = t.clone().view(-1, H, *t.shape[1:])
    t[:, [0, 1]] = t[:, [1, 0]]
    return t.view(-1, *t.shape[2:])


TEETH = {
    "include_key_len": ("o", "lse", "dq", "dk", "dv"),
    "drop_last_key_block": ("o", "lse", "dq", "dk", "dv"),
    "skip_alpha_rescale": ("o", "lse"),
    "scale_2^-7": ("o", "lse", "dq", "dk", "dv"),
    "swap_heads": ("o", "lse", "delta", "dq", "dk", "dv"),
    "no_dropout_rescale": ("o", "dq", "dk", "dv"),
    "delta_zero": ("delta", "dq", "dk"),
}


@pytest.mark.parametrize("fx", ["R0.7", "R2", "A-rise"])
@pytest.mark.parametrize("mutation", list(TEETH))
def test_bounds_have_teeth(fx, mutation):
    """The bound a correct kernel is held to is smaller than the mutation's effect on at least one
    element of every output it touches (fp64, padded S = 256, lengths 65 / 200 / 256, H = 2)."""
    c = Case("tiled", 256, (65, 200, 256), 2, fx, p=0.1 if mutation == "no_dropout_rescale" else 0.0)
    (q, k, v, do), kmask, _, n, S = case_data(c)
    q, k, v, do = heads(q), heads(k), heads(v), heads(do)
    zs, ds = None, 1.0
    if c.p:
        ds = dscale_of(c.p)
        zs = torch.from_numpy(attention_keep_ref(SEED, STEP + ADD, SITE, c.p, c.nseq, c.H, S)).to(F64) * ds
    r = ref_fwd(q, k, v, kmask, SCALE, zs)
    fb = fwd_bounds(q, k, v, kmask, SCALE, r, zs, ds)
    o_k, lse_k = bf(r["o"]), r["lse"]
    rb = ref_bwd(q, k, v, do, o_k, lse_k, kmask, SCALE, zs)
    bb = bwd_bounds(q, k, v, do, o_k, lse_k, kmask, SCALE, rb, zs, ds)
    ref = {"o": r["o"], "lse": r["lse"], **{x: rb[x] for x in ("delta", "dq", "dk", "dv")}}
    bound = {**fb, **bb}
    j = torch.arange(S)[None, :]
    nn_ = torch.tensor(n).repeat_interleave(c.H)[:, None]
    if mutation == "include_key_len":
        km2 = j <= nn_
        mf, mb = ref_fwd(q, k, v, km2, SCALE), ref_bwd(q, k, v, do, o_k, lse_k, km2, SCALE)
    elif mutation == "drop_last_key_block":
        km2 = j < 64 * ((nn_ + 63) // 64 - 1)
        mf, mb = ref_fwd(q, k, v, km2, SCALE), ref_bwd(q, k, v, do, o_k, lse_k, km2, SCALE)
    elif mutation == "skip_alpha_rescale":
        mf, mb = _skip_alpha(q, k, v, kmask, SCALE), {}
    elif mutation == "scale_2^-7":
        sc2 = SCALE * (1 + 2.0 ** -7)
        mf, mb = ref_fwd(q, k, v, kmask, sc2), ref_bwd(q, k, v, do, o_k, lse_k, kmask, sc2)
    elif mutation == "swap_heads":
        mf = {x: _swap(r[x], c.H) for x in ("o", "lse")}
        mb = {x: _swap(rb[x], c.H) for x in ("delta", "dq", "dk", "dv")}
    elif mutation == "no_dropout_rescale":
        mf = ref_fwd(q, k, v, kmask, SCALE, zs / ds)
        mb = ref_bwd(q, k, v, do, o_k, lse_k, kmask, SCALE, zs / ds)
    else:
        mb = dict(rb, delta=torch.zeros_like(rb["delta"]))
        P, dP = rb["P"], rb["dP"]
        dS = P * dP * SCALE
        mb["dq"], mb["dk"] = dS @ k, dS.mT @ q
        mf = {}
    mut = {**mf, **mb}
    for out in TEETH[mutation]:
        if (mutation, fx, out) == ("scale_2^-7", "R0.7", "dv"):
            continue      # a 0.8 % change of P on flat rows stays inside bf16(P)'s 2^-8: R2 shows it

        bad = violations(mut[out], ref[out], bound[out], bf16_out=out not in ("lse", "delta"))
        assert bool(bad.any()), f"{mutation} on {fx} invisible in {out}"


# ------------------------------------------------------------------------------ GPU cases
def _wide(rows, H, extra, fill, dtype=BF16):
    full = torch.full((rows, H * D + extra), fill, device="cuda", dtype=dtype)
    return full, full[:, :H * D]


def _same_bits(a, b):
    return torch.equal(a.view(torch.int16 if a.dtype == BF16 else torch.int32),
                       b.view(torch.int16 if b.dtype == BF16 else torch.int32))


def run_case(c):
    """Launch forward and backward through the binding on canary-filled buffers and return the
    raw buffers, the layout and the fp64 inputs (heads form, on the GPU)."""
    from bflc_demo_b200._native import C
    (q, k, v, do), kmask, qmask, n, S = case_data(c, "cuda")
    B, H = c.nseq, c.H
    packed = c.route == "packed"
    if packed:
        cu = [0]
        for x in c.lens:
            cu.append(cu[-1] + x)
        rows = cu[-1] + c.trail
    else:
        rows = B * S

    def lay(x, junk):
        if not packed:
            return x.reshape(B * S, H * D)
        parts = [x[b, :c.lens[b]].reshape(-1, H * D) for b in range(B)]
        parts.append(torch.full((c.trail, H * D), junk, device="cuda", dtype=F64))
        return torch.cat(parts)

    ins = {}
    for name, x in (("q", q), ("k", k), ("v", v), ("do", do)):
        full, view = _wide(rows, H, c.ld, 7.0)     # junk in the gap: reading it changes results
        view.copy_(lay(x, 100.0 if name == "k" else 3.0))
        ins[name] = (full, view)
    outs = {name: _wide(rows, H, c.ld, CANARY) for name in ("o", "dq", "dk", "dv")}
    nw = B * H * S
    lse = torch.full((nw + 64,), CANARY, device="cuda")
    delta = torch.full((nw + 64,), CANARY, device="cuda")
    drop = {}
    if c.p:
        step = torch.tensor([STEP], device="cuda", dtype=torch.int32)
        drop = dict(dropout_p=c.p, seed=SEED, step=step, step_add=ADD, site=SITE)
    iv = {x: ins[x][1] for x in ins}
    ov = {x: outs[x][1] for x in outs}
    if packed:
        cu_d = torch.tensor(cu, device="cuda", dtype=torch.int32)
        C().attention_packed_fwd(iv["q"], iv["k"], iv["v"], ov["o"], lse, cu_d, c.S, H, SCALE, **drop)
        C().attention_packed_bwd(iv["q"], iv["k"], iv["v"], ov["o"], iv["do"], lse, ov["dq"], ov["dk"], ov["dv"],
                                 delta, cu_d, c.S, H, SCALE, **drop)
    else:
        lengths = None if c.lens is None else torch.tensor(c.lens, device="cuda", dtype=torch.int32)
        C().attention_fwd(iv["q"], iv["k"], iv["v"], ov["o"], lse, B, S, H, SCALE, lengths, **drop)
        C().attention_bwd(iv["q"], iv["k"], iv["v"], ov["o"], iv["do"], lse, ov["dq"], ov["dk"], ov["dv"], B, S, H,
                          SCALE, delta, lengths, **drop)
    torch.cuda.synchronize()
    written = torch.zeros(rows, dtype=torch.bool, device="cuda")
    if packed:
        for b in range(B):
            written[cu[b]:cu[b] + n[b]] = True
    else:
        written[:] = True

    def unlay(t):
        x = t.to(F64)
        if not packed:
            return heads(x.view(B, S, H, D))
        out = torch.zeros(B, S, H, D, device="cuda", dtype=F64)
        for b in range(B):
            out[b, :n[b]] = x[cu[b]:cu[b] + n[b]].view(-1, H, D)
        return heads(out)

    return dict(q=heads(q), k=heads(k), v=heads(v), do=heads(do) * qmask[..., None], kmask=kmask, qmask=qmask,
                n=n, S=S, outs=outs, lse=lse, delta=delta, written=written, unlay=unlay, nw=nw)


def check_canaries(c, r):
    """Every element outside the written region still holds the NaN canary, bit for bit; every
    element inside it was written (is not NaN)."""
    H = c.H
    for name, (full, _) in r["outs"].items():
        region = torch.zeros_like(full, dtype=torch.bool)
        region[r["written"], :H * D] = True
        assert not bool(torch.isnan(full[region].float()).any()), f"{name}: unwritten element"
        canary = torch.full_like(full[~region], CANARY)
        assert _same_bits(full[~region], canary), f"{name}: written outside its rows / head columns"
    S, G = r["S"], c.nseq * H
    ln = torch.tensor(r["n"], device="cuda").repeat_interleave(H)[:, None]
    rows = torch.arange(S, device="cuda")[None, :]
    if c.route == "packed":
        live = rows < 64 * ((ln + 63) // 64)
    else:
        live = torch.ones(G, S, dtype=torch.bool, device="cuda")
    for name in ("lse", "delta"):
        buf = r[name]
        region = torch.zeros_like(buf, dtype=torch.bool)
        if name == "lse" or c.route != "whole":
            region[:r["nw"]] = live.reshape(-1)
        assert not bool(torch.isnan(buf[region]).any()), f"{name}: unwritten element"
        assert _same_bits(buf[~region], torch.full_like(buf[~region], CANARY)), f"{name}: canary overwritten"
    return live


@gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id())
def test_attention_case(case):
    c = case
    r = run_case(c)
    q, k, v, do, kmask, qmask = (r[x] for x in ("q", "k", "v", "do", "kmask", "qmask"))
    S = r["S"]
    G = c.nseq * c.H
    live = check_canaries(c, r)
    # route: the whole-route backward never writes delta (canary checked above); the tiled ones do
    o_k = r["unlay"](r["outs"]["o"][1])
    lse_k = r["lse"][:r["nw"]].view(G, S).to(F64)
    delta_k = r["delta"][:r["nw"]].view(G, S).to(F64)
    rowm = qmask[..., None]
    zs, ds = None, 1.0
    if c.p:
        ds = dscale_of(c.p)
        keep = attention_keep_ref(SEED, STEP + ADD, SITE, c.p, c.nseq, c.H, S)
        zs = torch.from_numpy(keep).to("cuda", F64) * ds
    nq_acc = 64 * torch.ceil(kmask.sum(-1).to(F64) / 64)[:, None, None] if c.route == "packed" else float(S)
    # ---- forward: O and lse against fp64
    rf = ref_fwd(q, k, v, kmask, SCALE, zs)
    fb = fwd_bounds(q, k, v, kmask, SCALE, rf, zs, ds)
    _report(violations(lse_k, rf["lse"], fb["lse"], bf16_out=False) & qmask, f"{c.id()} lse")
    exact = c.fx.startswith("E")
    if exact:
        e = exact_expectation(q, k, v, do, kmask, qmask, SCALE)
        _report((o_k != e["o"]) & rowm, f"{c.id()} O (exact)")
    else:
        _report(violations(o_k, rf["o"], fb["o"]) & rowm, f"{c.id()} O")
    # ---- backward: from the kernel's own O (bf16) and lse
    lse_in = torch.where(qmask, lse_k, 0.0)
    rb = ref_bwd(q, k, v, do, o_k * rowm, lse_in, kmask, SCALE, zs, qmask)
    grads = {x: r["unlay"](r["outs"][x][1]) for x in ("dq", "dk", "dv")}
    if c.route != "whole":
        if c.route == "packed":                     # rows past the length inside a live block: 0
            pad = live & ~qmask
            assert not bool(delta_k[pad].any()), f"{c.id()} delta past the length"
        if exact:
            _report((delta_k != e["delta"]) & qmask, f"{c.id()} delta (exact)")
    if exact:
        for x in ("dq", "dk", "dv"):
            _report((grads[x] != e[x]) & rowm, f"{c.id()} {x} (exact)")
        return
    bb = bwd_bounds(q, k, v, do, o_k * rowm, lse_in, kmask, SCALE, rb, zs, ds, qmask, nq_acc)
    if c.route != "whole":
        _report(violations(delta_k, rb["delta"], bb["delta"], bf16_out=False) & qmask, f"{c.id()} delta")
    for x in ("dq", "dk", "dv"):
        _report(violations(grads[x], rb[x], bb[x]) & rowm, f"{c.id()} {x}")
    if c.route == "tiled" and c.lens is not None:   # masked keys: exactly zero dK and dV
        for x in ("dk", "dv"):
            assert not bool(grads[x][~kmask].any()), f"{c.id()} {x} on masked keys"


@gpu
@pytest.mark.parametrize("family", ["whole", "tiled", "tiled-dropout", "packed", "packed-dropout"])
def test_public_ops_match_binding(family):
    """ops.nn.attention / attention_packed (forward and autograd backward) give bit-identical results
    to the direct binding calls on the same contiguous tensors."""
    from bflc_demo_b200._native import C
    from bflc_demo_b200.ops import nn as F
    H = 3
    p = 0.1 if family.endswith("dropout") else 0.0
    step = torch.tensor([STEP], device="cuda", dtype=torch.int32)
    rng = F.DropoutRNG(SEED, step, ADD)
    drop = dict(dropout_p=p, seed=SEED, step=step, step_add=ADD, site=SITE) if p else {}
    g = torch.Generator(device="cuda").manual_seed(1)
    if family.startswith("packed"):
        lens = (200, 0, 65, 1, 129)
        B, S, rows = len(lens), max(lens), sum(lens)
        cu = torch.tensor(np.cumsum((0,) + lens), device="cuda", dtype=torch.int32)
    else:
        B, S = 2, (128 if family == "whole" else 192)
        rows = B * S
        lengths = None if family == "whole" else torch.tensor([150, 7], device="cuda", dtype=torch.int32)
    q, k, v = [(torch.randn(rows, H * D, device="cuda", generator=g) * 0.7).to(BF16) for _ in range(3)]
    do = torch.randn(rows, H * D, device="cuda", generator=g).to(BF16)
    qa, ka, va = (t.clone().requires_grad_(True) for t in (q, k, v))
    if family.startswith("packed"):
        o = F.attention_packed(qa, ka, va, cu, S, H, dropout_p=p, rng=rng, site=SITE)
    else:
        o = F.attention(qa, ka, va, B, S, H, lengths=lengths, dropout_p=p, rng=rng, site=SITE)
    o.backward(do)
    o2, dq, dk, dv = (torch.empty_like(q) for _ in range(4))
    Sp = (S + 63) // 64 * 64
    lse, delta = (torch.empty(B * H * Sp, device="cuda") for _ in range(2))
    if family.startswith("packed"):
        C().attention_packed_fwd(q, k, v, o2, lse, cu, S, H, SCALE, **drop)
        C().attention_packed_bwd(q, k, v, o2, do, lse, dq, dk, dv, delta, cu, S, H, SCALE, **drop)
    else:
        C().attention_fwd(q, k, v, o2, lse, B, S, H, SCALE, lengths, **drop)
        C().attention_bwd(q, k, v, o2, do, lse, dq, dk, dv, B, S, H, SCALE,
                          None if family == "whole" else delta, lengths, **drop)
    torch.cuda.synchronize()
    for name, a, b in (("o", o.detach(), o2), ("dq", qa.grad, dq), ("dk", ka.grad, dk), ("dv", va.grad, dv)):
        assert _same_bits(a, b), name
