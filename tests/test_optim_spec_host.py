"""Exact specification of the flat optimizer kernels (``csrc/kernels/elementwise_optim.cu``): the four
``k_optim`` instantiations (plain / recipe x SGD / Adam), ``k_grad_norm`` and the cast / add helpers,
with every rounding point spelled out in numpy.  ``test_gpu_optim_conformance.py`` imports it.

What the build emits (``--use_fast_math``, sm_90a): every fp32 mul / add / sub / fma flushes
subnormal inputs and results to signed zero (``.ftz``); Adam's three divisions are
``div.approx.ftz`` (a multiply by an approximate reciprocal), ``sqrtf`` is ``sqrt.approx.ftz`` and
``powf`` is ``ex2.approx(lg2.approx(beta) * t)``; the bf16 casts are ``cvt.rn.bf16{x2}.f32``
(round to nearest even, subnormals kept).  So, per element and in the kernel's order:

* recipe only: ``g_in = coef * g`` (``__fmul_rn``), ``keep = 1 - lr_t * decay`` or 1 where the
  no-decay bit of 8-float block ``i >> 3`` is set, ``lr_t = f32(lr) * f32(f(t - 1))`` with f the
  schedule factor in fp64 exactly as ``lr_factor`` computes it;
* ``g = fma(wd, w, g_in)`` (coupled decay; 0 on the recipe path), then recipe ``w = w * keep``;
* SGD ``w = fma(-lr, g, w)``; Adam ``m = fma(b1, m, (1 - b1) * g)``,
  ``v = fma(b2, v, g * ((1 - b2) * g))`` -- all exact -- and
  ``w -= lr * (m / bc1) / (sqrt(v / bc2) + eps)``, ``bc = 1 - beta^t``, whose approximate
  operations get a derived bound (``adam_w_bound``);
* the bf16 shadow is the round-to-nearest-even of the kernel's own new ``w``; a zeroed gradient is +0.

``k_grad_norm``: ``norm = f32(sqrt(sum of exact fp64 squares))``, the squares of flushed inputs
(``cvt.ftz.f64.f32``: a subnormal gradient entry contributes 0); ``coef = min(1, f32(c) /
(norm + f32(1e-6)))`` exactly (``__fdiv_rn``, flushed below 2^-126); ``nonfinite = !isfinite(norm)``, which includes
finite gradients whose norm overflows fp32 (the recipe step is then skipped).

The CPU tests check the fp32 FMA against ``fractions.Fraction``, the specification (with flushing
off) against fp64 ``torch.optim`` + ``LambdaLR`` + ``clip_grad_norm_``, and that ten plausible kernel
mistakes each change a checked output of the GPU file's fixtures beyond its tolerance.
"""
from __future__ import annotations

import contextlib
import math
import os
import re
import shutil
import subprocess
from dataclasses import dataclass, replace
from fractions import Fraction
from typing import Optional

import numpy as np
import pytest

from test_gpu_trainer_conformance import pow_err

F32, F64 = np.float32, np.float64
TINY = 2.0 ** -126        # smallest normal fp32
U = 2.0 ** -24            # fp32 unit roundoff
ULP = 2.0 ** -23          # one fp32 ulp relative to the value
SH_INIT = 0x7FC1          # bf16 NaN the shadow holds before a launch: an element not written stays it
_FTZ = [True]


@contextlib.contextmanager
def no_ftz():
    """Evaluate the specification with IEEE subnormals (for the comparison with torch)."""
    _FTZ[0] = False
    try:
        yield
    finally:
        _FTZ[0] = True


def ftz(x):
    x = np.asarray(x, dtype=F32)
    if not _FTZ[0]:
        return x
    with np.errstate(invalid="ignore"):
        return np.where(np.abs(x) < TINY, x * F32(0), x)


def f32_mul(a, b):
    with np.errstate(over="ignore", invalid="ignore"):
        return ftz(ftz(a) * ftz(b))


def f32_add(a, b):
    with np.errstate(over="ignore", invalid="ignore"):
        return ftz(ftz(a) + ftz(b))


def f32_sub(a, b):
    with np.errstate(over="ignore", invalid="ignore"):
        return ftz(ftz(a) - ftz(b))


def f32_fma(a, b, c):
    """fp32 fma(a, b, c) rounded once: the product is exact in fp64, TwoSum gives the fp64 sum and
    its error, the sum is made round-to-odd from the error, and one rounding to fp32 follows (53 >=
    24 + 2 bits, so the round-to-odd intermediate cannot double-round)."""
    a, b, c = (np.broadcast_to(ftz(x), np.broadcast(a, b, c).shape).astype(F64) for x in (a, b, c))
    with np.errstate(over="ignore", invalid="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        err = (p - (s - bb)) + (c - bb)
        bits = s.view(np.int64)
        fix = np.isfinite(s) & np.isfinite(err) & (err != 0) & ((bits & 1) == 0)
        bits = np.where(fix, np.where(np.signbit(err) == np.signbit(s), bits + 1, bits - 1), bits)
        return ftz(bits.view(F64).astype(F32))


def bits32(x):
    return np.ascontiguousarray(x, dtype=F32).view(np.uint32)


def rne_bf16(x):
    """fp32 -> bf16 bits, round to nearest even; NaN -> a quiet NaN, overflow -> inf, subnormals kept."""
    b = bits32(x).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(np.asarray(x, F32)), ((b >> 16) | 0x40).astype(np.uint16), r)


def bf16_to_f32(h):
    return (np.asarray(h, np.uint16).astype(np.uint32) << 16).view(F32)


def same_bits(a, b):
    """Element-wise: identical fp32 bits, or both NaN."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    return (bits32(a) == bits32(b)) | (np.isnan(a) & np.isnan(b))


def same_bf16(a, b):
    a, b = np.asarray(a, np.uint16), np.asarray(b, np.uint16)
    return (a == b) | (np.isnan(bf16_to_f32(a)) & np.isnan(bf16_to_f32(b)))


def first_bad(ok, k=5):
    return np.flatnonzero(~np.asarray(ok))[:k].tolist()


# ------------------------------------------------------------------------------ schedule
LR_CONSTANT, LR_LINEAR, LR_COSINE = 0, 1, 2


def lr_factor64(schedule, W, T, s):
    """f(s) in fp64, operation for operation as the kernel's ``lr_factor`` (cospi -> cos(pi x))."""
    if s < W:
        return s / W
    if schedule == LR_CONSTANT:
        return 1.0
    span = float(max(1, T - W))
    if schedule == LR_LINEAR:
        return max(0.0, (T - s) / span)
    return max(0.0, 0.5 * (1.0 + math.cos(math.pi * ((s - W) / span))))


def lr_t(lr, schedule, W, T, s):
    f = lr_factor64(schedule, W, T, s)
    if schedule == LR_COSINE and s >= W:
        # cospi on the device and cos(pi x) here differ by ulps of fp64: no fp32 rounding boundary
        # may lie that close, or the fixture must pick another step
        assert F32(f * (1 - 2.0 ** -40)) == F32(f * (1 + 2.0 ** -40)), (s, W, T, f)
    return f32_mul(F32(lr), ftz(F32(f)))


# ------------------------------------------------------------------------------ the update
@dataclass
class Case:
    adam: bool
    n: int
    w: np.ndarray
    g: np.ndarray
    m: np.ndarray
    v: np.ndarray
    lr: float
    step: int
    word: Optional[int]                 # device step word (None: no step word)
    zero_grad: bool
    wd: float = 0.0                     # coupled decay (plain optim_step only)
    b1: float = 0.9
    b2: float = 0.999
    eps: float = 1e-8
    recipe: bool = False
    schedule: int = LR_CONSTANT
    W: int = 0
    T: int = 0
    decay: float = 0.0
    mask: Optional[np.ndarray] = None   # int32 no-decay words
    clip: Optional[str] = None          # None | "header" | "norm" (workspace given)
    coef: float = 1.0
    nonfinite: int = 0
    label: str = ""

    @property
    def t(self):
        return (self.word or 0) + self.step


def _keep(c, dec, mutant):
    i = np.arange(c.n, dtype=np.int64)
    blk = i >> 3
    if mutant == "nodecay_block_i_gt_2":          # vector body: float4 index >> 2 instead of >> 1
        nv = c.n // 4 * 4
        blk = np.where(i < nv, i >> 4, blk)
    if c.mask is None:
        bit = np.zeros(c.n, dtype=bool)
    else:
        words = c.mask.view(np.uint32).astype(np.uint64)
        bit = ((words[blk >> 5] >> (blk & 31).astype(np.uint64)) & 1).astype(bool)
    return np.where(bit, F32(1), f32_sub(F32(1), dec)).astype(F32)


def run_update(c: Case, mutant: Optional[str] = None):
    """The update of ``c`` as the kernel computes it.  Exact outputs, and for Adam the weight entering
    the last line (``w_pre``) plus the centre of its bound as ``w``.  ``mutant`` names a kernel
    mistake to model instead (the teeth test)."""
    n = c.n
    w0, g0 = c.w.astype(F32), c.g.astype(F32)
    out = {"grad": np.zeros(n, F32) if c.zero_grad else g0.copy()}
    if c.recipe and c.clip is not None and c.nonfinite:
        out.update(w=w0.copy(), m=c.m.copy(), v=c.v.copy(), shadow=None, skipped=True)
        return out
    t = c.step if mutant == "step_word_ignored" else c.t
    b1, b2 = F32(c.b1), F32(c.b2)
    if mutant == "betas_swapped":
        b1, b2 = b2, b1
    if c.recipe:
        s = t if mutant == "lr_from_f_t" else t - 1
        lr = lr_t(c.lr, c.schedule, c.W, c.T, s)
        keep = _keep(c, f32_mul(lr, F32(c.decay)), mutant)
        coef = F32(1) if (c.clip is None or mutant == "coef_not_applied") else F32(c.coef)
        g_in = f32_mul(coef, g0)
        wd = F32(0)
    else:
        lr, keep, g_in, wd = F32(c.lr), None, g0, F32(c.wd)
    g = f32_fma(wd, w0, g_in)
    w = f32_mul(w0, keep) if (keep is not None and mutant != "decay_after_update") else ftz(w0)
    if c.adam:
        m = f32_fma(b1, c.m, f32_mul(f32_sub(F32(1), b1), g))
        v = f32_fma(b2, c.v, f32_mul(g, f32_mul(f32_sub(F32(1), b2), g)))
        tb = t - 1 if mutant == "bias_correction_t_minus_1" else t
        wn = adam_w_centre(w, m, v, lr, b1, b2, F32(c.eps), tb, eps_in_sqrt=mutant == "eps_inside_sqrt")
        out.update(m=m, v=v, w_pre=w)
    else:
        wn = f32_fma(-lr, g, w)
        out.update(m=c.m.copy(), v=c.v.copy())
    if keep is not None and mutant == "decay_after_update":
        wn = f32_mul(wn, keep)
    out.update(w=wn, lr=lr, t=t, skipped=False)
    out["shadow"] = rne_bf16(w0 if mutant == "shadow_from_old_w" else wn)
    if mutant == "tail_drops_last" and n % 4:
        for k in ("w", "m", "v"):
            out[k][-1] = {"w": c.w, "m": c.m, "v": c.v}[k][-1]
        out["shadow"][-1] = SH_INIT
        out["grad"][-1] = g0[-1]
    return out


def adam_w_centre(w, m, v, lr, b1, b2, eps, t, eps_in_sqrt=False):
    """fp32 rounding of the fp64 Adam line on the kernel's operands (inside adam_w_bound)."""
    b1, b2 = float(b1), float(b2)
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    with np.errstate(all="ignore"):
        m64, v64 = m.astype(F64), v.astype(F64)
        den = np.sqrt(v64 / bc2 + float(eps)) if eps_in_sqrt else np.sqrt(v64 / bc2) + float(eps)
        return ftz((w.astype(F64) - float(lr) * (m64 / bc1) / den).astype(F32))


def adam_w_bound(w_pre, m, v, lr, b1, b2, eps, t):
    """Reference (fp64) and tolerance of Adam's last line from the kernel's own m', v' and t.

    bc = 1 - __powf(beta, t): pow_err absolute, plus one rounding of 1 - p unless Sterbenz makes it
    exact (p >= 1/2).  m' / bc1 and v' / bc2: a multiply by an approximate reciprocal, 2 ulp each;
    sqrt.approx 1 ulp; + eps, * lr and the final w - x: one rounding each, which the bound allows to
    be fused or not (ptxas folds w - a * rcp(d) into one FFMA); the last division 2 ulp.  Flushing:
    lr * m / bc1 below 2^-126 drops the whole update, a flushed v / bc2 moves s by at most
    2^-63, and the result itself may flush (2^-126)."""
    b1, b2, lr, eps = float(b1), float(b2), float(lr), float(eps)
    w0, m, v = (np.asarray(x, F32).astype(F64) for x in (w_pre, m, v))
    p1, p2 = b1 ** t, b2 ** t
    bc1, bc2 = 1 - p1, 1 - p2
    r1 = (pow_err(b1, t) + (U * bc1 if p1 < 0.5 else 0.0)) / bc1
    r2 = (pow_err(b2, t) + (U * bc2 if p2 < 0.5 else 0.0)) / bc2
    with np.errstate(all="ignore"):
        A = m / bc1
        q = v / bc2
        s = np.sqrt(q)
        D = s + eps
        upd = lr * A / D
        ref = w0 - upd
        rA = r1 / (1 - r1) + 2 * ULP + U                         # m * rcp(bc1), then * lr
        rs = (r2 / (1 - r2) + 2 * ULP) / 2 + ULP + 2.0 ** -63 / np.maximum(s, 2.0 ** -200)
        rD = rs * s / D + U
        R = (rA + rD / (1 - rD) + 2 * ULP + U) * (1 + 1e-3)
        tol = np.abs(upd) * R + U * np.abs(ref) + 2 * TINY
        lost = (np.abs(lr * A) < 2 * TINY) | (q > 3.0e38)      # flushed numerator / overflowed radicand
        tol = np.where(lost, tol + np.abs(upd), tol)
    return ref, tol


def check_update(c: Case, out: dict, spec: Optional[dict] = None):
    """Failures of a launch's outputs (numpy: w, m, v, grad fp32; shadow bf16 bits) against the
    specification of ``c``; empty when conformant."""
    sp = spec if spec is not None else run_update(c)
    bad = []

    def need(name, ok):
        ok = np.asarray(ok)
        if not ok.all():
            bad.append(f"{c.label} {name}: {int((~ok).sum())} of {ok.size} differ, first at {first_bad(ok)}")

    need("grad", same_bits(out["grad"], sp["grad"]))
    if sp["skipped"]:
        for k, ref in (("w", c.w), ("m", c.m), ("v", c.v)):
            if k == "w" or c.adam:
                need(k, same_bits(out[k], ref))
        need("shadow", out["shadow"] == SH_INIT)
        return bad
    if c.adam:
        need("m", same_bits(out["m"], sp["m"]))
        need("v", same_bits(out["v"], sp["v"]))
        ref, tol = adam_w_bound(sp["w_pre"], out["m"], out["v"], sp["lr"], c.b1, c.b2, F32(c.eps), sp["t"])
        w = out["w"].astype(F64)
        with np.errstate(invalid="ignore"):
            need("w (bound)", (np.abs(w - ref) <= tol) | (w == ref) | (np.isnan(w) & np.isnan(ref)))
    else:
        need("w", same_bits(out["w"], sp["w"]))
    need("shadow = rne(w)", same_bf16(out["shadow"], rne_bf16(out["w"])))
    return bad


# ------------------------------------------------------------------------------ gradient norm
def grad_norm_spec(g):
    """(norm, ambiguous): the kernel's fp32 norm, and whether the exact norm lies within the fp64
    summation error n 2^-53 of an fp32 rounding boundary (then 1 ulp either way is conformant)."""
    g64 = ftz(g).astype(F64)
    if np.isnan(g64).any():
        return F32(np.nan), False
    if np.isinf(g64).any():
        return F32(np.inf), False
    N = math.sqrt(math.fsum((g64 * g64).tolist()))
    d = (len(g64) + 2) * 2.0 ** -53
    with np.errstate(over="ignore"):
        return ftz(F32(N)), bool(F32(N * (1 - d)) != F32(N * (1 + d)))


def clip_spec(norm, c):
    """(coef, nonfinite) of the workspace header from the kernel's fp32 norm."""
    norm = F32(norm)
    if not np.isfinite(norm):
        return F32(1), 1
    with np.errstate(over="ignore"):
        return min(F32(1), ftz(F32(c) / f32_add(norm, F32(1e-6)))), 0      # div.rn.ftz: may flush


# ------------------------------------------------------------------------------ casts
def cast_u8_spec(u, scale):
    return rne_bf16(f32_mul(np.asarray(u, np.uint8).astype(F32), F32(scale)))


def add_bf16_spec(a_bits, b_bits):
    return rne_bf16(f32_add(bf16_to_f32(a_bits), bf16_to_f32(b_bits)))


# ------------------------------------------------------------------------------ fixtures
BF16_TIES = [0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000, 0x7F7F8000]


def _edge_pairs(nonfinite):
    tie = bits_f32(BF16_TIES)
    e = [(tie[0], 0.0), (tie[1], 0.0), (tie[2], 0.0), (tie[3], 0.0),   # shadow ties: g = 0 keeps w
         (0.0, 0.0), (-0.0, -0.0), (1e-40, 0.5), (0.5, 1e-40), (-1e-39, -3e-39),
         (1.0, 1e-25), (-2.0, -1e-25),                                  # g^2 underflows: v -> 0
         (1.0, 1e30), (-3.0, -1e30)]                                    # g^2 overflows: v -> inf
    if nonfinite:
        e += [(1.0, np.nan), (1.0, np.inf), (-1.0, -np.inf)]
    return e


def bits_f32(bits):
    return np.asarray(bits, np.uint32).view(F32)


def values(n, seed, nonfinite=False, moments=True):
    """w, g, m, v: normal values at several scales (g ~ 1e-6 makes eps matter), with the edge pairs
    at the front and again at the back (the tail loop), as far as n allows."""
    rng = np.random.default_rng(seed)
    w = (rng.standard_normal(n) * rng.choice([1.0, 1e-3, 1e3], n)).astype(F32)
    gs = rng.choice([1.0, 1e-6, 1e-3, 10.0], n)
    g = (rng.standard_normal(n) * gs).astype(F32)
    e = _edge_pairs(nonfinite)
    k = min(len(e), n)
    pos = list(range(k)) + (list(range(n - k, n)) if n >= 2 * k else [])
    for j, p in enumerate(pos):
        w[p], g[p] = e[j % len(e)]
    if moments:
        m = (rng.standard_normal(n) * gs * 0.3).astype(F32)
        v = (np.square(rng.standard_normal(n) * gs) * 0.5).astype(F32)
    else:
        m, v = np.zeros(n, F32), np.zeros(n, F32)
    return w, g, m, v


def random_mask(n, seed):
    words = np.random.default_rng(seed).integers(0, 2 ** 32, (n + 255) // 256, dtype=np.uint64).astype(np.uint32)
    last = (n - 1) >> 3                                  # the block holding the tail
    words[last >> 5] |= np.uint32(1 << (last & 31))
    words[0] |= np.uint32(1 << 31)
    return words.view(np.int32)


N_OPT = [1, 3, 4, 5, 8, 9, 255, 257, 4099, 100004, 1081344 + 13]
STEPS = [(1, None), (3, 0), (1, 1000), (2, 1 << 20)]


def plain_cases(adam, n):
    out = []
    for j, (wd, (step, word), zg) in enumerate((wd, st, zg) for wd in (0.0, 0.1) for st in STEPS
                                               for zg in (True, False)):
        if n > 200000 and j % 3:
            continue
        w, g, m, v = values(n, 1000 * j + n % 997, nonfinite=True, moments=(step, word) != (1, None))
        out.append(Case(adam, n, w, g, m, v, lr=1.23e-2 if adam else 0.0873, step=step, word=word, zero_grad=zg,
                        wd=wd, label=f"plain {'adam' if adam else 'sgd'} n={n} wd={wd} t=({step},{word}) zg={zg}"))
    return out


RECIPE_W, RECIPE_T = 3, 10
RECIPE_T_STEPS = [2, 4, 6, 11, 13]          # s = t - 1 below, at and above W; at and above T


def recipe_cases(adam, n):
    out = []
    clips = [None, "header", None, "header"]
    for j, (sched, t) in enumerate((sc, t) for sc in (LR_CONSTANT, LR_LINEAR, LR_COSINE) for t in RECIPE_T_STEPS):
        if n > 200000 and j % 3:
            continue
        w, g, m, v = values(n, 7000 + 100 * j + n % 997, moments=t > 1)
        step, word = (t, None) if j % 2 else (1, t - 1)
        decay = 0.1 if j % 2 == 0 else 0.0
        out.append(Case(adam, n, w, g, m, v, lr=2.1e-2 if adam else 0.173, step=step, word=word,
                        zero_grad=j % 3 != 2, recipe=True, schedule=sched, W=RECIPE_W, T=RECIPE_T, decay=decay,
                        mask=random_mask(n, j) if decay or j % 4 == 1 else None, clip=clips[j % 4],
                        coef=0.375, label=f"recipe {'adam' if adam else 'sgd'} n={n} sched={sched} t={t} "
                                          f"decay={decay} clip={clips[j % 4]}"))
    return out


def teeth_cases():
    cs = plain_cases(True, 257)[:8] + plain_cases(False, 257)[:4] + recipe_cases(True, 4099) + \
        recipe_cases(False, 257)
    return cs


MUTANTS = ["bias_correction_t_minus_1", "nodecay_block_i_gt_2", "decay_after_update", "coef_not_applied",
           "eps_inside_sqrt", "betas_swapped", "lr_from_f_t", "shadow_from_old_w", "tail_drops_last",
           "step_word_ignored"]


# ============================================================================== CPU tests
def _frac_fma(a, b, c):
    return Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))


def _round_f32(q: Fraction):
    """Round a rational to fp32, nearest even (normal range), by bracketing with numpy neighbours."""
    x = F32(float(q))                       # within one ulp
    lo, hi = (np.nextafter(x, F32(-np.inf)), x) if Fraction(float(x)) > q else (x, np.nextafter(x, F32(np.inf)))
    dl, dh = q - Fraction(float(lo)), Fraction(float(hi)) - q
    if dl != dh:
        return lo if dl < dh else hi
    return lo if (bits32(lo) & 1) == 0 else hi


def test_fma_matches_fractions_on_random_triples():
    rng = np.random.default_rng(1)
    a = (rng.standard_normal(3000) * 2.0 ** rng.integers(-20, 20, 3000)).astype(F32)
    b = (rng.standard_normal(3000) * 2.0 ** rng.integers(-20, 20, 3000)).astype(F32)
    c = (-(a.astype(F64) * b) * (1 + rng.standard_normal(3000) * 2.0 ** -rng.integers(1, 40, 3000))).astype(F32)
    got = f32_fma(a, b, c)
    for i in range(3000):
        q = _frac_fma(a[i], b[i], c[i])
        want = F32(0) if q == 0 else _round_f32(q)
        if abs(float(want)) < TINY:
            want = F32(0.0) if q >= 0 else F32(-0.0)
        assert bits32(got[i]) == bits32(want) or (q == 0 and got[i] == 0), (i, a[i], b[i], c[i], got[i], want)


def _midpoint_triples():
    """a * b + c whose fp64 sum lands exactly on an fp32 midpoint although the exact value does not:
    c has an odd last bit, a * b = half an ulp of c minus 2^-46 of it."""
    rng = np.random.default_rng(2)
    out = []
    for _ in range(200):
        e = int(rng.integers(-60, 60))
        c = F32((1 + (2 * int(rng.integers(0, 2 ** 22)) + 1) * 2.0 ** -23) * 2.0 ** e)
        sgn = float(rng.choice([-1.0, 1.0]))
        a, b = F32(1 + 2.0 ** -23), F32((1 - 2.0 ** -23) * 2.0 ** (e - 24) * sgn)
        out.append((a, b, F32(c * sgn)))
    return out


def test_fma_is_single_rounding_where_the_naive_form_double_rounds():
    naive_wrong = 0
    for a, b, c in _midpoint_triples():
        want = _round_f32(_frac_fma(a, b, c))
        assert bits32(f32_fma(a, b, c)) == bits32(want), (a, b, c)
        naive = F32(F64(a) * F64(b) + F64(c))
        naive_wrong += int(bool((bits32(naive) != bits32(want)).any()))
    assert naive_wrong == 200


def test_ftz_primitives_flush_inputs_and_results_to_signed_zero():
    assert bits32(f32_mul(F32(1e-40), F32(1e10))) == 0
    assert bits32(f32_mul(F32(-1e-20), F32(1e-20))) == 0x80000000
    assert bits32(f32_add(F32(-1e-40), F32(-0.0))) == 0x80000000
    assert bits32(f32_fma(F32(1e-20), F32(1e-20), F32(-1e-40))) == 0
    assert f32_fma(F32(2.0), F32(3.0), F32(1e-40)) == 6.0
    with no_ftz():
        assert f32_mul(F32(1e-40), F32(2.0)) == F32(1e-40) * F32(2.0) != 0


def test_rne_bf16_matches_torch():
    import torch
    rng = np.random.default_rng(3)
    x = rng.integers(0, 2 ** 32, 200000, dtype=np.uint64).astype(np.uint32).view(F32)
    x = np.concatenate([x, bits_f32(BF16_TIES), np.array([np.inf, -np.inf, 0.0, -0.0, 3.4e38, 1e-45], F32)])
    ref = torch.from_numpy(x.copy()).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    assert same_bf16(rne_bf16(x), ref).all()


def test_lr_factor_is_the_host_mirror_and_cosine_fixtures_are_unambiguous():
    from bflc_demo_b200.ops.optim import lr_factor
    for sched, name in ((0, "constant"), (1, "linear"), (2, "cosine")):
        for s in range(0, 16):
            # ops.optim rounds pi * (s - W) before dividing; the kernel takes cospi((s - W) / span)
            assert lr_factor64(sched, RECIPE_W, RECIPE_T, s) == pytest.approx(lr_factor(name, s, RECIPE_W, RECIPE_T),
                                                                              rel=1e-15, abs=1e-15)
            lr_t(0.173, sched, RECIPE_W, RECIPE_T, s)                    # asserts no boundary nearby
    assert lr_t(0.173, LR_LINEAR, RECIPE_W, RECIPE_T, 10) == 0 and lr_t(0.173, LR_LINEAR, 3, 10, 0) == 0


def test_grad_norm_spec():
    g = np.array([3.0, 4.0], F32)
    assert grad_norm_spec(g) == (F32(5.0), False)
    assert grad_norm_spec(np.array([1e-40, 3.0], F32))[0] == 3.0              # subnormals flushed
    assert np.isnan(grad_norm_spec(np.array([1.0, np.nan, np.inf], F32))[0])
    assert np.isinf(grad_norm_spec(np.array([3e38, 3e38], F32))[0])             # finite, overflows
    assert clip_spec(np.inf, 1.0) == (1.0, 1) and clip_spec(F32(5.0), 1.0)[0] == F32(1.0) / F32(5.000001)
    assert clip_spec(F32(0.5), 1.0)[0] == 1.0


def _torch_steps(kind, w0, grads, lr, wd, sched=None, clip=None, mask_groups=None):
    import torch
    p = torch.nn.Parameter(torch.from_numpy(w0.astype(F64)))
    if mask_groups is not None:
        dec, nod = mask_groups
        ps = [torch.nn.Parameter(torch.from_numpy(w0[i].astype(F64))) for i in (dec, nod)]
        groups = [{"params": [ps[0]], "weight_decay": wd}, {"params": [ps[1]], "weight_decay": 0.0}]
    else:
        ps, groups = [p], [{"params": [p], "weight_decay": wd}]
    opt = {"sgd": torch.optim.SGD, "adam": torch.optim.Adam, "adamw": torch.optim.AdamW}[kind]
    kw = {} if kind == "sgd" else dict(betas=(0.9, 0.999), eps=1e-8)
    o = opt(groups, lr=lr, foreach=False, **kw)
    sch = torch.optim.lr_scheduler.LambdaLR(o, sched) if sched else None
    for gk in grads:
        for q, idx in zip(ps, mask_groups or [slice(None)]):
            q.grad = torch.from_numpy(gk[idx].astype(F64))
        if clip:
            torch.nn.utils.clip_grad_norm_(ps, clip)
        o.step()
        if sch:
            sch.step()
    out = np.zeros(len(w0), F64)
    for q, idx in zip(ps, mask_groups or [slice(None)]):
        out[idx] = q.detach().numpy()
    return out


@pytest.mark.parametrize("kind", ["sgd", "adam", "recipe_sgd", "recipe_adamw"])
def test_spec_without_ftz_is_torch_fp64(kind):
    """The specification is the right algorithm, not the kernel restated: with IEEE subnormals it
    follows fp64 torch.optim (+ LambdaLR + clip_grad_norm_ for the recipe) to within fp32 rounding."""
    n, steps, rng = 1000, 4, np.random.default_rng(9)
    w0 = rng.standard_normal(n).astype(F32)
    grads = [(rng.standard_normal(n) * 0.3).astype(F32) for _ in range(steps)]
    adam = "adam" in kind
    lr = 1e-2 if adam else 0.1
    mask = random_mask(n, 4)
    blk = np.arange(n) >> 3
    nod = ((mask.view(np.uint32)[blk >> 5] >> (blk & 31).astype(np.uint32)) & 1).astype(bool)
    w, m, v = w0.copy(), np.zeros(n, F32), np.zeros(n, F32)
    with no_ftz():
        for k, gk in enumerate(grads):
            c = Case(adam, n, w, gk, m, v, lr=lr, step=k + 1, word=None, zero_grad=True)
            if kind.startswith("recipe"):
                norm, _ = grad_norm_spec(gk)
                c = replace(c, recipe=True, schedule=LR_LINEAR, W=2, T=10, decay=0.1, mask=mask, clip="norm",
                            coef=clip_spec(norm, 1.0)[0])
            else:
                c = replace(c, wd=0.1)
            o = run_update(c)
            w, m, v = o["w"], o["m"], o["v"]
    if kind.startswith("recipe"):
        ref = _torch_steps("adamw" if adam else "sgd", w0, grads, lr, 0.1,
                           sched=lambda s: lr_factor64(LR_LINEAR, 2, 10, s), clip=1.0,
                           mask_groups=(np.flatnonzero(~nod), np.flatnonzero(nod)))
    else:
        ref = _torch_steps("adam" if adam else "sgd", w0, grads, lr, 0.1)
    delta = np.abs(ref - w0)
    err = np.abs(w.astype(F64) - ref)
    assert (err <= 2e-5 * delta + steps * 2 * U * np.abs(ref) + 1e-12).all(), first_bad(
        err <= 2e-5 * delta + steps * 2 * U * np.abs(ref) + 1e-12)


def test_kernel_model_conforms_on_the_gpu_fixtures():
    for c in teeth_cases():
        o = run_update(c)
        if c.adam and not o["skipped"]:
            assert np.isfinite(o["w"]).sum() > 0
        assert check_update(c, o) == [], c.label


@pytest.mark.parametrize("mutant", MUTANTS)
def test_teeth_every_kernel_mistake_fails_a_fixture(mutant):
    """Each modelled kernel mistake changes at least one checked output of the GPU file's fixtures
    beyond its exact or bounded tolerance."""
    caught = [c.label for c in teeth_cases() if check_update(c, run_update(c, mutant), spec=run_update(c))]
    assert caught, mutant


def test_optimizer_and_norm_kernels_spill_free(tmp_path):
    from bflc_demo_b200 import build
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("no nvcc")
    inc = [f"-I{build.CSRC / d}" for d in ("include", "ledger", "runtime")]
    src = build.CSRC / "kernels" / "elementwise_optim.cu"
    proc = subprocess.run([nvcc, *build.GENCODE, *build.NVCC_FLAGS, *inc, "-c", str(src), "-o", str(tmp_path / "e.o")],
                          capture_output=True, text=True, timeout=900)
    log = proc.stdout + proc.stderr
    assert proc.returncode == 0, log[-3000:]
    props = re.findall(r"Function properties for (\w+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    found = {n: tuple(map(int, r)) for n, *r in props if "k_optim" in n or "k_grad_norm" in n}
    assert len(found) == 5, log[-3000:]
    for name, v in found.items():
        assert v == (0, 0, 0), (name, v)
