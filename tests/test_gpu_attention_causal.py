"""Conformance of the causal fused attention kernels (``attn_causal_{fwd,dq,dkv}`` in
``csrc/kernels/attn_sm100.cu``) against float64, element by element.

The method is ``test_gpu_attention_conformance.py``'s, with the key mask generalised to a mask per
(query, key): ``mask[g, i, j]`` = key j is visible to query i (causal: j <= i).  The reference and
the rounding-model bounds below are that suite's ``ref_fwd`` / ``ref_bwd`` / ``fwd_bounds`` /
``bwd_bounds`` with every per-head quantity (valid key count, key blocks, row max) taken per query
row: under the causal mask query row i reads the ceil((i + 1) / 64) key blocks up to its diagonal.
The forward is checked on O and lse; the backward on delta, dQ, dK and dV from the kernel's own O and
lse, so a forward error is never charged to the backward.  Every output is a column slice of a
wider NaN-filled buffer (and lse / delta have NaN tails): each canary outside the written region
must survive.

Exact fixtures (the ex2 argument of every non-target score is <= -128, so it flushes to 0):
* ``E1-diag``: key j scores 1024 j for every query, so row i's maximum is its diagonal key: O = V
  row by row, bit for bit.  Admitting key i + 1 would give V[i + 1].
* ``E1-first``: key j scores -1024 j: every row picks key 0, O = V[0].
* ``E1-spread`` (S = 64): one-hot key codes, row i targets key (7 i) mod (i + 1).
* ``E2`` ties: keys 2m and 2m + 1 score alike, so an odd row splits 1/2 : 1/2 between its diagonal
  and the key before it, and an even row, whose tie partner lies past the diagonal, takes V[i] alone.
With P one-hot or exact halves and small-integer V and dO, O and dV are exact dyadic sums, and with
one-hot P dQ = dK = 0.  ``E1-diag`` stays at S <= 320: its row maximum 1024 i times scale log2e
reaches 2^16 near row 355, where one rounding of that product (2^-8) moves p off 1 before P is
rounded to bf16 -- a score range far outside attention's, which the rounding model does not cover.
"""
import math

import pytest
import torch

from test_dropout_host import attention_keep_ref
from test_gpu_attention_conformance import (BF16, BF_U, D, EX2, F32, F64, FTZ, LOG2E, LOGF_ABS, LOGF_REL, RCP,
                                            SCALE, U, ULP, _report, dscale_of, gamma, violations)

gpu = pytest.mark.gpu
SEED, STEP, ADD, SITE = 0x0123_4567_89AB_CDEF, 9, 2, 5
NAN = float("nan")


# ----------------------------------------------------------------------- float64 reference
def causal_mask(G, S):
    return torch.ones(S, S, dtype=torch.bool).tril().expand(G, S, S)


def ref_fwd(q, k, v, mask, scale, zs=None):
    s = q @ k.mT
    x = (scale * s).masked_fill(~mask, -math.inf)
    lse = torch.logsumexp(x, -1)
    P = torch.exp(x - lse[..., None])
    W = P if zs is None else P * zs
    return {"s": s, "P": P, "o": W @ v, "lse": lse}


def ref_bwd(q, k, v, do, o, lse, mask, scale, zs=None):
    s = q @ k.mT
    P = torch.exp((scale * s - lse[..., None]).masked_fill(~mask, -math.inf))
    delta = (do * o).sum(-1)
    dP = do @ v.mT
    Gd = dP if zs is None else zs * dP
    dS = P * (Gd - delta[..., None]) * scale
    W = P if zs is None else P * zs
    return {"P": P, "dP": dP, "G": Gd, "dS": dS, "delta": delta, "dq": dS @ k, "dk": dS.mT @ q, "dv": W.mT @ do,
            "s": s}


def fwd_bounds(q, k, v, mask, scale, ref, zs=None, dscale=1.0):
    """``test_gpu_attention_conformance.fwd_bounds`` with the key count n, the key blocks and the row
    max taken per query row."""
    s, P = ref["s"], ref["P"]
    es = gamma(D) * (q.abs() @ k.abs().mT)
    m = s.masked_fill(~mask, -math.inf).amax(-1, keepdim=True)
    esm = es.masked_fill(~mask, 0).amax(-1, keepdim=True)
    sc = scale * LOG2E
    x = ((s - m) * sc).masked_fill(~mask, 0).abs()
    dx = sc * (es + esm) * (1 + U) + 4 * U * x
    rp = (torch.exp2(dx) * (1 + EX2) - 1).masked_fill(~mask, 0)
    n = mask.sum(-1, keepdim=True).to(F64)
    nkb = torch.ceil(n / 64)
    g = 1 + gamma(64 * nkb)
    chain = (1 + ULP) ** nkb
    rpm = rp.amax(-1, keepdim=True)
    rl = (1 + rpm) * g * chain - 1
    rest = (1 + BF_U) * g * chain * (1 + RCP) * (1 + U) * (1 + (U if zs is not None else 0))
    rw = (1 + rp) * rest / (1 - rl) - 1
    W = P if zs is None else P * zs
    ob = (W * rw) @ v.abs() + FTZ * dscale * (mask.to(F64) @ v.abs())
    ra = (torch.exp2(4 * U * x.amax(-1, keepdim=True)) * (1 + EX2)) ** nkb
    el = (1 + rpm) * g * chain * ra - 1 + n * FTZ
    lse = ref["lse"][..., None]
    lb = (scale * esm * (1 + U) - torch.log1p(-el) + LOGF_ABS
          + LOGF_REL * (torch.log(n) + el) + 2 * U * (scale * m.abs() + lse.abs() + 1))
    return {"o": ob, "lse": lb[..., 0]}


def bwd_bounds(q, k, v, do, o, lse, mask, scale, ref, zs=None, dscale=1.0):
    """``test_gpu_attention_conformance.bwd_bounds`` with the dQ accumulation length per query row."""
    vf = mask.to(F64)
    n = mask.sum(-1, keepdim=True).to(F64)
    nk_acc = 64 * torch.ceil(n / 64)
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


# ----------------------------------------------------------------------------- fixtures
def fixture(name, B, S, H, seed=0):
    """q, k, v, dO as fp64 heads [G, S, 64] holding bf16 values."""
    G = B * H
    g = torch.Generator().manual_seed(seed)
    j = torch.arange(S, dtype=F64)
    v = torch.randint(-8, 9, (G, S, D), generator=g).to(F64)
    do = torch.randint(-4, 5, (G, S, D), generator=g).to(F64)
    q = torch.zeros(G, S, D, dtype=F64)
    k = torch.zeros(G, S, D, dtype=F64)
    if name in ("E1-diag", "E1-first"):              # score 1024 (j - i) (or -1024 j), exact in fp32
        k[..., 0], k[..., 1] = torch.div(j, 64, rounding_mode="floor"), j % 64
        sign = 1.0 if name == "E1-diag" else -1.0
        q[..., 0], q[..., 1] = sign * 65536.0, sign * 1024.0

    elif name == "E1-spread":                        # S = 64: one-hot codes, target (7 i) mod (i + 1)
        assert S == 64
        k[:, torch.arange(S), torch.arange(S)] = 8.0
        t = (7 * torch.arange(S)) % (torch.arange(S) + 1)
        q[:, torch.arange(S), t] = 128.0
    elif name == "E2":                               # keys 2m, 2m + 1 score 1024 m
        c = torch.div(j, 2, rounding_mode="floor")
        k[..., 0], k[..., 1] = torch.div(c, 32, rounding_mode="floor"), c % 32
        q[..., 0], q[..., 1] = 32 * 1024.0, 1024.0

    elif name == "A-rise":                           # the row max rises in every key block (alpha < 1)
        q = 0.5 * torch.randn(G, S, D, generator=g, dtype=F64)
        k = 0.5 * torch.randn(G, S, D, generator=g, dtype=F64)
        k[..., 0], q[..., 0] = 0.05 * j, 8.0
        v, do = torch.randn(G, S, D, generator=g, dtype=F64), torch.randn(G, S, D, generator=g, dtype=F64)
    else:                                            # R<scale>: realistic
        sc = {"R": 0.7, "R2": 2.0}[name]
        q, k = (sc * torch.randn(G, S, D, generator=g, dtype=F64) for _ in range(2))
        v, do = torch.randn(G, S, D, generator=g, dtype=F64), torch.randn(G, S, D, generator=g, dtype=F64)
    return tuple(t.to(BF16).to(F64) for t in (q, k, v, do))


def exact_expect(name, v, do, S):
    """O and dV of the exact fixtures (P one-hot or exact halves)."""
    G = v.shape[0]
    i = torch.arange(S)
    if name == "E1-diag":
        W = torch.eye(S, dtype=F64)
    elif name == "E1-first":
        W = torch.zeros(S, S, dtype=F64)
        W[:, 0] = 1
    elif name == "E1-spread":
        W = torch.zeros(S, S, dtype=F64)
        W[i, (7 * i) % (i + 1)] = 1
    else:
        W = torch.eye(S, dtype=F64)
        odd = i[1::2]
        W[odd, odd] = 0.5
        W[odd, odd - 1] = 0.5
    W = W.expand(G, S, S)
    return W @ v, W.mT @ do


def to_rows(x, B, H, S):
    """heads [B*H, S, 64] -> [B*S, H*64]"""
    return x.view(B, H, S, D).permute(0, 2, 1, 3).reshape(B * S, H * D)


def heads(x, B, H, S):
    return x.reshape(B, S, H, D).permute(0, 2, 1, 3).reshape(B * H, S, D)


def _wide(rows, cols, extra, fill=NAN, dtype=BF16):
    return torch.full((rows, cols + extra), fill, device="cuda", dtype=dtype)


def run(B, S, H, q, k, v, do, extra, p=0.0):
    """Runs the causal kernels on wide NaN-filled buffers -> (buffers, slices)."""
    from bflc_demo_b200._native import C
    rows, cols = B * S, H * D
    bufs = {n: _wide(rows, cols, extra) for n in ("q", "k", "v", "do", "o", "dq", "dk", "dv")}
    for n, t in (("q", q), ("k", k), ("v", v), ("do", do)):
        bufs[n][:, :cols] = to_rows(t, B, H, S).to(BF16).cuda()
    sl = {n: b[:, :cols] for n, b in bufs.items()}
    lse = torch.full((B * H * S + 32,), NAN, device="cuda")
    delta = torch.full_like(lse, NAN)
    kw = {}
    if p > 0:
        step = torch.tensor([STEP], device="cuda", dtype=torch.int32)
        kw = dict(dropout_p=p, seed=SEED, step=step, step_add=ADD, site=SITE)
    C().attention_fwd(sl["q"], sl["k"], sl["v"], sl["o"], lse, B, S, H, SCALE, None, causal=True, **kw)
    C().attention_bwd(sl["q"], sl["k"], sl["v"], sl["o"], sl["do"], lse, sl["dq"], sl["dk"], sl["dv"], B, S, H,
                      SCALE, delta, None, causal=True, **kw)
    torch.cuda.synchronize()
    return bufs, sl, lse, delta


def check_canaries(bufs, cols, lse, delta, n):
    for name in ("o", "dq", "dk", "dv"):
        gap = bufs[name][:, cols:]
        assert torch.isnan(gap.float()).all(), f"{name}: a write past the head columns"
        assert not torch.isnan(bufs[name][:, :cols].float()).any(), f"{name}: an element left unwritten"
    for name, t in (("lse", lse), ("delta", delta)):
        assert torch.isnan(t[n:]).all(), f"{name}: a write past B*H*S"
        assert torch.isfinite(t[:n]).all(), f"{name}: an element left unwritten"


def check_case(B, S, H, fx, extra=0, p=0.0, seed=0):
    q, k, v, do = fixture(fx, B, S, H, seed)
    bufs, sl, lse, delta = run(B, S, H, q, k, v, do, extra, p)
    n = B * H * S
    check_canaries(bufs, H * D, lse, delta, n)
    G = B * H
    mask = causal_mask(G, S)
    zs, dsc = None, 1.0
    if p > 0:
        dsc = dscale_of(p)
        keep = torch.from_numpy(attention_keep_ref(SEED, STEP + ADD, SITE, p, B, H, S))
        zs = keep.to(F64) * dsc
    o_k = heads(sl["o"].cpu().to(F64), B, H, S)
    lse_k = lse[:n].cpu().to(F64).view(G, S)
    ref = ref_fwd(q, k, v, mask, SCALE, zs)
    fb = fwd_bounds(q, k, v, mask, SCALE, ref, zs, dsc)
    _report(violations(o_k, ref["o"], fb["o"]), f"{fx} O")
    _report(violations(lse_k, ref["lse"], fb["lse"], bf16_out=False), f"{fx} lse")
    rb = ref_bwd(q, k, v, do, o_k, lse_k, mask, SCALE, zs)
    bb = bwd_bounds(q, k, v, do, o_k, lse_k, mask, SCALE, rb, zs, dsc)
    _report(violations(delta[:n].cpu().to(F64).view(G, S), rb["delta"], bb["delta"], bf16_out=False),
            f"{fx} delta")
    for name in ("dq", "dk", "dv"):
        out = heads(sl[name].cpu().to(F64), B, H, S)
        _report(violations(out, rb[name], bb[name]), f"{fx} {name}")
    if fx.startswith("E") and p == 0:
        o_x, dv_x = exact_expect(fx, v, do, S)
        assert torch.equal(o_k, o_x), f"{fx}: O differs from the exact rows"
        assert torch.equal(heads(sl["dv"].cpu().to(F64), B, H, S), dv_x), f"{fx}: dV inexact"
        if fx.startswith("E1"):                      # one-hot P: dS = P (dP - delta) = 0 exactly
            for name in ("dq", "dk"):
                assert torch.count_nonzero(sl[name].float()) == 0, f"{fx}: {name} should be exactly 0"
    return bufs


# ---------------------------------------------------------------------------- CPU guards
def test_reference_matches_sdpa_is_causal():
    B, S, H = 2, 128, 3
    q, k, v, do = fixture("R", B, S, H, seed=4)
    G = B * H
    ref = ref_fwd(q, k, v, causal_mask(G, S), SCALE)
    qa, ka, va = (t.clone().requires_grad_(True) for t in (q, k, v))
    o = torch.nn.functional.scaled_dot_product_attention(qa, ka, va, is_causal=True, scale=SCALE)
    assert torch.allclose(o, ref["o"], atol=1e-12, rtol=1e-12)
    o.backward(do)
    rb = ref_bwd(q, k, v, do, ref["o"], ref["lse"], causal_mask(G, S), SCALE)
    for name, t in (("dq", qa), ("dk", ka), ("dv", va)):
        assert torch.allclose(t.grad, rb[name], atol=1e-10, rtol=1e-10), name


@pytest.mark.parametrize("fx,S", [("E1-diag", 320), ("E1-first", 320), ("E1-spread", 64), ("E2", 448)])
def test_exact_fixture_premises(fx, S):
    q, k, v, do = fixture(fx, 1, S, 2)
    ref = ref_fwd(q, k, v, causal_mask(2, S), SCALE)
    o_x, dv_x = exact_expect(fx, v, do, S)
    assert ((ref["o"] - o_x).abs() <= 1e-9).all()     # fp64 rounding and the (unflushed) tiny weights
    s = (ref["s"] * SCALE * LOG2E).masked_fill(~causal_mask(2, S), -math.inf)
    top = s.amax(-1, keepdim=True)
    second = s.masked_fill(s >= top, -math.inf).amax(-1)
    gap = (top[..., 0] - second)[:, 1:]               # row 0 has a single visible key
    assert (gap >= 128).all()                         # every non-target p flushes to exactly 0


MUTATIONS = ("admit_next", "drop_diag")


@pytest.mark.parametrize("mutation", MUTATIONS)
@pytest.mark.parametrize("fx", ["R", "A-rise"])
def test_bounds_have_teeth(fx, mutation):
    """Admitting key i + 1 or dropping the diagonal key breaks the bounds on at least one element of
    O, lse, dQ, dK and dV."""
    B, S, H = 1, 192, 2
    q, k, v, do = fixture(fx, B, S, H, seed=3)
    G = B * H
    mask = causal_mask(G, S)
    ref = ref_fwd(q, k, v, mask, SCALE)
    fb = fwd_bounds(q, k, v, mask, SCALE, ref)
    i = torch.arange(S)
    bad = mask.clone()
    if mutation == "admit_next":
        bad[:, i[:-1], i[:-1] + 1] = True
    else:
        bad[:, i[1:], i[1:]] = False
    wrong = ref_fwd(q, k, v, bad, SCALE)
    assert violations(wrong["o"], ref["o"], fb["o"]).any()
    assert violations(wrong["lse"], ref["lse"], fb["lse"], bf16_out=False).any()
    rb = ref_bwd(q, k, v, do, ref["o"], ref["lse"], mask, SCALE)
    bb = bwd_bounds(q, k, v, do, ref["o"], ref["lse"], mask, SCALE, rb)
    wb = ref_bwd(q, k, v, do, ref["o"], ref["lse"], bad, SCALE)
    for name in ("dq", "dk", "dv"):
        assert violations(wb[name], rb[name], bb[name]).any(), name


# ----------------------------------------------------------------------------------- GPU
SS = (64, 128, 192, 256, 320, 384, 448, 512)
BH = ((1, 1), (3, 4), (1, 12))


@gpu
@pytest.mark.parametrize("B,H", BH)
@pytest.mark.parametrize("S", SS)
def test_causal_realistic(S, B, H):
    check_case(B, S, H, "R", seed=S + H)


@gpu
@pytest.mark.parametrize("fx,S", [("E1-diag", 320), ("E1-diag", 192), ("E1-first", 320), ("E1-spread", 64),
                                  ("E2", 448), ("E2", 128), ("A-rise", 512), ("R2", 384)])
def test_causal_fixtures(fx, S):
    check_case(3, S, 4, fx, extra=72)


@gpu
def test_causal_wide_pitch():
    check_case(3, 256, 12, "R", extra=72, seed=11)


@gpu
@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("S", [64, 128, 512])
def test_causal_dropout(S, p):
    check_case(3, S, 4, "R", extra=72, p=p, seed=int(p * 10) + S)


@gpu
def test_causal_bit_identical_runs():
    q, k, v, do = fixture("R", 3, 384, 4, seed=5)
    a = run(3, 384, 4, q, k, v, do, 0)
    b = run(3, 384, 4, q, k, v, do, 0)
    for name in ("o", "dq", "dk", "dv"):
        assert torch.equal(a[1][name].view(torch.int16), b[1][name].view(torch.int16)), name
    n = 3 * 4 * 384
    assert torch.equal(a[2][:n], b[2][:n]) and torch.equal(a[3][:n], b[3][:n])


@gpu
def test_routing_and_rejected_combinations():
    """Causal S = 128 runs the tiled kernels (they write delta; the one-CTA-per-head backward never
    does), ops.nn forwards the flag, and every unsupported combination is refused."""
    from bflc_demo_b200._native import C
    from bflc_demo_b200.ops import nn as F
    B, S, H = 2, 128, 2
    q, k, v, do = fixture("R", B, S, H, seed=9)
    _, _, _, delta = run(B, S, H, q, k, v, do, 0)
    assert torch.isfinite(delta[:B * H * S]).all()
    qr, kr, vr = (to_rows(t, B, H, S).to(BF16).cuda().requires_grad_(True) for t in (q, k, v))
    o = F.attention(qr, kr, vr, B, S, H, causal=True)
    o.backward(to_rows(do, B, H, S).to(BF16).cuda())
    bufs, sl, _, _ = run(B, S, H, q, k, v, do, 0)
    assert torch.equal(o.detach(), sl["o"]) and torch.equal(qr.grad, sl["dq"]) and torch.equal(vr.grad, sl["dv"])
    lengths = torch.full((B,), S, device="cuda", dtype=torch.int32)
    with pytest.raises(ValueError):
        F.attention(qr, kr, vr, B, S, H, causal=True, lengths=lengths)
    with pytest.raises(ValueError):
        F.attention(qr, kr, vr, B, S, H, causal=True, fused=False)
    with pytest.raises(ValueError):
        F.attention(qr[:, :96], kr[:, :96], vr[:, :96], B, S, 1, causal=True)     # head dim 96
    cu = torch.tensor([0, S, 2 * S], device="cuda", dtype=torch.int32)
    with pytest.raises(ValueError):
        F.attention_packed(qr, kr, vr, cu, S, H, causal=True)
    out = torch.empty_like(sl["o"])
    lse = torch.empty(B * H * S, device="cuda")
    with pytest.raises(RuntimeError, match="not supported"):
        C().attention_fwd(sl["q"], sl["k"], sl["v"], out, lse, B, S, H, SCALE, lengths, causal=True)
