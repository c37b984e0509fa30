"""Conformance of the persistent MLP trainer (``csrc/kernels/mlp_round_sm100.cu``, driven through
``models/mlp.py::FlatMLP.train_epoch_fused``) against a plain float64 reference of the training step
defined here: forward, softmax cross-entropy, both weight gradients, the hidden gradient, the bias
column sums and the SGD / Adam update.

* One step, every stage.  Each stage is checked against fp64 computed from the kernel's own upstream
  bf16 intermediates (``h``, ``h_dq``, ``dlogits``, ``dh``), so per-element bounds stay tight and an
  error is pinned to the stage that made it.  The weight gradients are consumed by the optimizer, so
  they are checked through the update of the fp32 master (and the Adam moments).
* Several steps in one launch against the same steps as single-step launches, bit for bit, on a
  saturated fixture whose bias column sums are exact in any order.

Two kinds of comparison, as in ``test_gpu_layer_conformance.py`` (whose helpers are reused):

* exact -- the integer fixture: x in {0, 1}, W1 / W2 in {-1, 0, 1}, integer b1 and b2 = integer +
  a distinct multiple of 1/1024 per class.  h is an integer below 256 and every logit is exact in
  fp32 and tie-free, so h and ``correct`` equal the fp64 reference.
* bound -- ``|out - ref| <= derived slack + half an ulp of out's type``.  Products of bf16 values
  are exact in fp32, so a GEMM differs from exact arithmetic only by its fp32 sums: with
  u = 2^-23 (one fp32 ulp per addition, which also covers truncating accumulation, in any order)
  a sum of n terms is within gamma_n * sum |terms|, gamma_n = n u / (1 - n u).  The build uses
  --use_fast_math; the CUDA C++ Programming Guide bounds the functions that replace: __expf
  within 2 + floor(1.173 |x|) ulp, __logf within 2^-21.41 absolute on [0.5, 2] and 3 ulp
  elsewhere, x / y within 2 ulp, sqrtf within 1 ulp, __powf as exp2f(y * __log2f(x)) with exp2f
  within 2 ulp and __log2f within 2^-22 absolute on [0.5, 2].

Every GPU case asserts from the kernel's %globaltimer stamps which phase plan and optimizer
placement ran, and states the weight-gradient tile height the launcher's rule picks on this device.
The fp64 self-check of the reference and the fixture guards run on the CPU.
"""
import math
from typing import NamedTuple

import pytest
import torch

from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec, sf_bytes
from bflc_demo_b200.ops.mx8 import quantize_mx8_reference
from test_gpu_layer_conformance import assert_bound, assert_exact

gpu = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24            # fp32 unit roundoff (one rounding to nearest)
ULP = 2.0 ** -23          # one fp32 ulp, relative to the value
# FlatMLP's Adam constants as the kernel holds them (fp32)
BETA1, BETA2, EPS = (float(torch.tensor(v, dtype=F32)) for v in (0.9, 0.999, 1e-8))
LR = {"sgd": 0.05, "adam": 1e-3}
DEFAULT_PLAN = 4


def f32(v):
    return float(torch.tensor(v, dtype=F32))


def gamma(n):
    return n * ULP / (1 - n * ULP)


def rne_bf16(t):
    return t.to(F32).to(BF16).double()


# ----------------------------------------------------------------------- float64 reference
def softmax_xent(z, y, B):
    """Per-row softmax cross-entropy of fp64 logits z [R, C]: probabilities, dlogits = (p - onehot)
    / B, per-row loss."""
    zmax = z.amax(1, keepdim=True)
    e = torch.exp(z - zmax)
    s = e.sum(1, keepdim=True)
    p = e / s
    onehot = torch.nn.functional.one_hot(y.long(), z.shape[1]).to(z.dtype)
    loss = (torch.log(s) + zmax).squeeze(1) - z.gather(1, y.long()[:, None]).squeeze(1)
    return p, (p - onehot) / B, loss


def ref_step(w1, b1, w2, b2, x, y):
    """One training step of the MLP in fp64: every intermediate and gradient of the mean loss."""
    B = x.shape[0]
    h = torch.relu(x @ w1.t() + b1)
    z = h @ w2.t() + b2
    p, dl, loss = softmax_xent(z, y, B)
    dh = (dl @ w2) * (h > 0)
    return {"h": h, "z": z, "dlogits": dl, "loss_sum": loss.sum(), "dh": dh,
            "correct": int((z.argmax(1) == y.long()).sum()),
            "w1": dh.t() @ x, "b1": dh.sum(0), "w2": dl.t() @ h, "b2": dl.sum(0)}


def sgd(w, g, lr):
    return w - lr * g


def adam(w, m, v, g, lr, tt):
    """Adam with bias correction from the step count tt, as the kernel writes it."""
    m = BETA1 * m + (1 - BETA1) * g
    v = BETA2 * v + (1 - BETA2) * g * g
    bc1, bc2 = 1 - BETA1 ** tt, 1 - BETA2 ** tt
    return w - lr * (m / bc1) / (torch.sqrt(v / bc2) + EPS), m, v


# ---------------------------------------------------------------- derived rounding bounds
def softmax_slack(z, ez, y, B):
    """Bound on |kernel's fp32 dlogits - fp64 dlogits| given logits within ez of z (per element).

    Logit errors of at most D = max_c ez in a row move every p_c by at most a factor exp(+-2D).  The
    kernel's t_c = z_c - vmax (one rounding), __expf(t_c) (2 + 1.173 |t_c| ulp), the fp32 sum of C
    positive terms (gamma_C), 1 / sum (2 ulp) and the product (one rounding) add relative errors;
    an underflowed exponential adds 2^-126.  Then p - onehot and * (1 / B) (2 ulp) round once each."""
    C = z.shape[1]
    _, dl, _ = softmax_xent(z, y, B)
    p = torch.softmax(z, 1)
    D = ez.amax(1, keepdim=True)
    t = (z - z.amax(1, keepdim=True)).abs() + 2 * D
    r = torch.expm1(2 * D) + U * t + (2 + 1.173 * t) * ULP + gamma(C) + 2 * ULP + U
    sp = p * r * (1 + r) + 2.0 ** -126
    v = (dl * B).abs()
    return ((sp * (1 + U) + U * (v + sp)) * (1 + 2 * ULP) + (U + 2 * ULP) * v) / B * (1 + 1e-6)


def pow_err(beta, tt):
    """Absolute error of __powf(beta, tt) = exp2f(tt * __log2f(beta)), beta in [0.5, 2]."""
    p = beta ** tt
    y = abs(tt * math.log2(beta))
    return p * (math.log(2) * (tt * 2.0 ** -22 + U * y) * (1 + 1e-6) + 2 * ULP)


def adam_slack(w0, m0, v0, g, sg, lr, tt):
    """fp64 Adam update of (w0, m0, v0) by gradient g and the bounds on the kernel's m', v', w' when
    its gradient lies within sg of g: the fp32 moment updates (at most three roundings), the
    bias corrections (__powf, then 1 - p: exact by Sterbenz for p >= 1/2, one rounding otherwise),
    the two approximate divisions, sqrtf, + eps, the last division, * lr and w - update.  Each
    product may also flush to zero (--use_fast_math implies -ftz): 2^-126 per product, which
    matters where lr * (m / bc1) falls below it and the update vanishes."""
    c1, c2 = 1 - BETA1, 1 - BETA2
    m = BETA1 * m0 + c1 * g
    v = BETA2 * v0 + c2 * g * g
    bc1, bc2 = 1 - BETA1 ** tt, 1 - BETA2 ** tt
    ftz = 2.0 ** -126
    sm = c1 * sg + 2 * U * (BETA1 * m0.abs() + c1 * g.abs()) + 2 * ftz
    sv = c2 * (2 * g.abs() * sg + sg * sg) + 3 * U * (BETA2 * v0 + c2 * g * g) + 3 * ftz
    e1 = pow_err(BETA1, tt) + (U * bc1 if BETA1 ** tt < 0.5 else 0.0)
    e2 = pow_err(BETA2, tt) + (U * bc2 if BETA2 ** tt < 0.5 else 0.0)
    r1, r2 = e1 / bc1, e2 / bc2
    A = m / bc1
    s = torch.sqrt(v / bc2)
    D = s + EPS
    upd = lr * A / D
    w = w0 - upd
    dA = sm / bc1 * (1 + r1) + A.abs() * (r1 + 2 * ULP) * (1 + 1e-6)
    arg_err = sv / bc2 * (1 + r2) + (v / bc2) * (r2 + 2 * ULP) * (1 + 1e-6)
    lin = arg_err / (2 * s).clamp_min(1e-300)
    ds = torch.minimum(torch.sqrt(arg_err), lin) + s * ULP
    dD = (ds + U * D) * (1 + 1e-6)
    Dlo = (D - dD).clamp_min(EPS * (1 - 1e-6))
    dU = (lr * (dA / Dlo + A.abs() * dD / (D * Dlo)) * (1 + 2 * U) + upd.abs() * (2 * ULP + 2 * U)
          + 2 * ftz / Dlo)
    return (w, m, v), (dU + U * w.abs(), sm, sv)


# ------------------------------------------------------------------------------- fixtures
class Fixture(NamedTuple):
    kind: str                # "int" | "real" | "sat"
    D: int
    H: int
    C: int
    B: int
    S: int
    master: torch.Tensor     # fp32 flat parameters (CPU)
    xu8: torch.Tensor        # uint8 [S*B, D]; x = bf16(xu8 / 255)
    y: torch.Tensor          # int32 [S*B]


def int_fixture(D, H, C, B, seed):
    """x in {0, 1} (every eighth row all zero), W1 / W2 in {-1, 0, 1}, b1 integer, b2 = integer + a
    distinct multiple of 1/1024 per class.  Hidden unit 0 has W1 row 0 = 0 and b1 = 4, and W2
    column 0 = -1: a zero row of x has h = (4, 0, ...) and logits b2 - 4 < 0, all negative.  Zero
    rows are labelled with their argmax, half of the others too."""
    g = torch.Generator().manual_seed(seed)
    spec = mlp_spec(D, H, C)
    master = torch.zeros(spec.total)
    v = spec.views(master)
    x = (torch.rand(B, D, generator=g) < 0.25).float()
    x[7::8] = 0
    w1 = torch.randint(-1, 2, (H, D), generator=g).float()
    w1[0] = 0
    b1 = torch.randint(-4, 1, (H,), generator=g).float()
    b1[0] = 4
    w2 = torch.randint(-1, 2, (C, H), generator=g).float()
    w2[:, 0] = -1
    b2 = torch.randint(-3, 4, (C,), generator=g).float() + torch.randperm(128, generator=g)[:C].float() / 1024
    v["w1"].copy_(w1)
    v["b1"].copy_(b1)
    v["w2"].copy_(w2)
    v["b2"].copy_(b2)
    z = torch.relu(x.double() @ w1.double().t() + b1.double()) @ w2.double().t() + b2.double()
    top = z.argmax(1).int()
    rnd = torch.randint(0, C, (B,), generator=g, dtype=torch.int32)
    keep = (torch.rand(B, generator=g) < 0.5) | (x.sum(1) == 0)
    y = torch.where(keep, top, rnd)
    return Fixture("int", D, H, C, B, 1, master, (x * 255).to(torch.uint8), y)


def real_fixture(D, H, C, B, seed):
    """spec.init_ weights, small random biases, u8-like inputs ((rand^2) * 255), random labels."""
    g = torch.Generator().manual_seed(seed)
    spec = mlp_spec(D, H, C)
    master = torch.empty(spec.total)
    spec.init_(master, seed=seed)
    v = spec.views(master)
    v["b1"].copy_(0.05 * torch.randn(H, generator=g))
    v["b2"].copy_(0.05 * torch.randn(C, generator=g))
    xu8 = (torch.rand(B, D, generator=g) ** 2 * 255).to(torch.uint8)
    y = torch.randint(0, C, (B,), generator=g, dtype=torch.int32)
    return Fixture("real", D, H, C, B, 1, master, xu8, y)


def sat_fixture(B, S, seed, D=784, H=256, C=62):
    """Every row's top logit leads by far more than 104: row r of class k(r) has x[r, k] = 1 over
    u8 noise below 0.1; hidden unit j of block j % C has W1[j, j % C] = 8 over U(-0.05, 0.05) noise;
    W2[c, j] = 7.5 on c's own block and +-0.75 elsewhere.  __expf of every other logit minus the top
    one underflows to 0, so dlogits is 0 or +-1/B, and the bias column sums are exact in any order
    (sat_guard checks both along an emulation of the whole trajectory)."""
    g = torch.Generator().manual_seed(seed)
    spec = mlp_spec(D, H, C)
    master = torch.zeros(spec.total)
    v = spec.views(master)
    k = torch.randint(0, C, (B * S,), generator=g)
    xu8 = torch.randint(0, 26, (B * S, D), generator=g).to(torch.uint8)
    xu8[torch.arange(B * S), k] = 255
    j = torch.arange(H)
    w1 = (torch.rand(H, D, generator=g) - 0.5) * 0.1
    w1[j, j % C] += 8
    w2 = torch.where(torch.rand(C, H, generator=g) < 0.5, 0.75, -0.75)
    w2[j % C, j] = 7.5
    v["w1"].copy_(w1)
    v["w2"].copy_(w2)
    rnd = torch.randint(0, C, (B * S,), generator=g)
    y = torch.where(torch.rand(B * S, generator=g) < 0.5, k, rnd).int()
    return Fixture("sat", D, H, C, B, S, master, xu8, y)


def x_bf16(fx):
    return (fx.xu8.float() * f32(1 / 255)).to(BF16)


def mx8_dq(t):
    return quantize_mx8_reference(t.float()).dequantize().double()


def dyadic_bits(terms):
    """Significant bits any partial sum (any order, any subset of rows) of each column of `terms`
    [rows, cols] can need: all terms are multiples of their lowest set bit 2^-k, and every partial
    sum is a multiple of it no larger than the column's sum of magnitudes."""
    s = terms * 2.0 ** 40
    assert torch.equal(s, s.round()), "terms off the 2^-40 grid"
    iv = s.round().to(torch.int64)
    nz = iv[iv != 0]
    if nz.numel() == 0:
        return 0
    low = int((nz & -nz).abs().min())
    total = int(iv.abs().sum(0).max())
    return math.ceil(math.log2(total / low + 1))


def sat_guard(fx, fp8, opt, base=0, rows=None, carry=None):
    """Emulates training steps on the fixture in fp64 on the kernel's operands (bf16 shadows, bf16 h;
    fp8: the quantiser's dequantised x, W and h) and asserts, at every step: the top-1 margin is at least
    104 with room for the emulation's own rounding (the kernel's logits are within ~1e-3 of it),
    so dlogits is 0 or +-1/B; every db1 / db2 column partial sum lies on a dyadic grid with fewer
    than 24 significant bits; |W2| stays in [0.5, 8].

    ``rows``: the row slice of each step (default: the fixture's S batches in order).  Adam's step
    count of step s is base + s + 1.  ``carry``: a dict {"p", "m", "v"} of fp64 parameter / moment
    views the steps start from and are left in (default: the fixture's model, zero moments)."""
    B, C = fx.B, fx.C
    spec = mlp_spec(fx.D, fx.H, fx.C)
    if carry is None:
        carry = {}
    if "p" not in carry:
        carry["p"] = {k: t.double().clone() for k, t in spec.views(fx.master).items()}
        carry["m"] = {k: torch.zeros_like(t) for k, t in carry["p"].items()}
        carry["v"] = {k: torch.zeros_like(t) for k, t in carry["p"].items()}
    p, m, vv = carry["p"], carry["m"], carry["v"]
    if rows is None:
        rows = [slice(s * B, (s + 1) * B) for s in range(fx.S)]
    lo, hi = min(r.start for r in rows), max(r.stop for r in rows)
    xb = torch.zeros(hi, fx.D, dtype=F64)
    xb[lo:hi] = x_bf16(fx._replace(xu8=fx.xu8[lo:hi])).double()
    xq = xb
    if fp8:
        xq = torch.zeros_like(xb)
        xq[lo:hi] = mx8_dq(fx.xu8[lo:hi].float() * f32(1 / 255))
    margins = []
    for s, r in enumerate(rows):
        w1s, w2s = rne_bf16(p["w1"]), rne_bf16(p["w2"])
        w1f, w2f = (mx8_dq(p["w1"]), mx8_dq(p["w2"])) if fp8 else (w1s, w2s)
        h = rne_bf16(torch.relu(xq[r] @ w1f.t() + p["b1"]))
        hin = mx8_dq(h) if fp8 else h
        z = hin @ w2f.t() + p["b2"]
        top2 = z.topk(2, dim=1)
        margin = float((top2.values[:, 0] - top2.values[:, 1]).min())
        margins.append(margin)
        assert margin >= 112, (s, margin)
        y = fx.y[r].long()
        dl = (torch.nn.functional.one_hot(top2.indices[:, 0], C) - torch.nn.functional.one_hot(y, C)).double() / B
        dh = (dl @ w2s) * (hin > 0)
        assert dyadic_bits(dl) < 24 and dyadic_bits(dh) < 24, s
        g = {"w1": rne_bf16(dh).t() @ xb[r], "b1": dh.sum(0), "w2": dl.t() @ h, "b2": dl.sum(0)}
        for k in p:
            if opt == "sgd":
                p[k] = sgd(p[k], g[k], LR[opt])
            else:
                p[k], m[k], vv[k] = adam(p[k], m[k], vv[k], g[k], LR[opt], base + s + 1)
        a = p["w2"].abs()
        assert float(a.min()) >= 0.5 and float(a.max()) <= 8, s
    return margins


# ------------------------------------------------------------------------------ CPU tests
def test_reference_matches_autograd_and_torch_optim():
    g = torch.Generator().manual_seed(3)
    B, D, H, C = 48, 40, 24, 10
    x = torch.rand(B, D, generator=g, dtype=F64)
    y = torch.randint(0, C, (B,), generator=g, dtype=torch.int32)
    params = {"w1": torch.randn(H, D, generator=g, dtype=F64) * 0.3, "b1": torch.randn(H, generator=g, dtype=F64) * 0.1,
              "w2": torch.randn(C, H, generator=g, dtype=F64) * 0.3, "b2": torch.randn(C, generator=g, dtype=F64) * 0.1}
    r = ref_step(params["w1"], params["b1"], params["w2"], params["b2"], x, y)
    leaf = {k: t.clone().requires_grad_(True) for k, t in params.items()}
    h = torch.relu(x @ leaf["w1"].t() + leaf["b1"])
    z = h @ leaf["w2"].t() + leaf["b2"]
    loss = torch.nn.functional.cross_entropy(z, y.long(), reduction="sum")
    loss.backward()
    assert abs(float(loss) - float(r["loss_sum"])) <= 1e-12 * float(loss)
    assert r["correct"] == int((z.argmax(1) == y.long()).sum())
    for k in params:
        assert torch.allclose(leaf[k].grad / B, r[k], rtol=1e-12, atol=1e-15), k
    for lr, opt in ((0.05, "sgd"), (1e-3, "adam")):
        for base in (0, 7):
            ps = [params[k].clone().requires_grad_(True) for k in params]
            m0 = [torch.randn(t.shape, generator=g, dtype=F64) * 1e-2 * (base > 0) for t in ps]
            v0 = [torch.rand(t.shape, generator=g, dtype=F64) * 1e-4 * (base > 0) for t in ps]
            if opt == "sgd":
                o = torch.optim.SGD(ps, lr=lr)
            else:
                o = torch.optim.Adam(ps, lr=lr, betas=(BETA1, BETA2), eps=EPS)
                for t, m, v in zip(ps, m0, v0):
                    o.state[t] = {"step": torch.tensor(float(base)), "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
            for t, k in zip(ps, params):
                t.grad = r[k].clone()
            o.step()
            for t, k, m, v in zip(ps, params, m0, v0):
                want = (sgd(params[k], r[k], lr) if opt == "sgd" else adam(params[k], m, v, r[k], lr, base + 1)[0])
                assert torch.allclose(t.detach(), want, rtol=1e-13, atol=1e-16), (opt, base, k)


def test_reference_tt_is_visible():
    """The Adam bound resolves an off-by-one step count at the tt the suite uses."""
    g = torch.Generator().manual_seed(5)
    w0 = torch.randn(4096, generator=g, dtype=F64) * 0.05
    m0 = torch.randn(4096, generator=g, dtype=F64) * 1e-3
    v0 = torch.rand(4096, generator=g, dtype=F64) * 1e-6
    gr = torch.randn(4096, generator=g, dtype=F64) * 1e-3
    for tt in (1, 8):
        (w, m, v), (sw, sm, sv) = adam_slack(w0, m0, v0, gr, gr.abs() * 1e-5, 1e-3, tt)
        w_off = adam(w0, m0, v0, gr, 1e-3, tt + 1)[0]
        assert bool(((w_off - w).abs() > sw + 2 * U * w.abs()).any()), tt


@pytest.mark.parametrize("D,H,C,B", [(784, 256, 62, 512), (784, 256, 64, 256), (784, 256, 10, 256),
                                     (512, 256, 62, 256), (64, 256, 62, 128), (784, 128, 62, 200),
                                     (784, 640, 62, 128), (784, 256, 62, 2048)])
def test_int_fixture_is_exact(D, H, C, B):
    """h is an integer below 256; logits are exact in fp32 (|z| < 2^13 on the 2^-10 grid) and
    tie-free, both from h and from the quantiser's dequantised h (fp8: fwd2 reads h_dq); some
    rows have only negative logits and are hits."""
    fx = int_fixture(D, H, C, B, seed=D + H + C + B)
    v = {k: t.double() for k, t in mlp_spec(D, H, C).views(fx.master).items()}
    x = x_bf16(fx).double()
    assert torch.equal(x, fx.xu8.double() / 255)
    h = torch.relu(x @ v["w1"].t() + v["b1"])
    assert torch.equal(h, h.round()) and float(h.max()) < 256
    for hin in (h, mx8_dq(h)):
        z = hin @ v["w2"].t() + v["b2"]
        assert float(z.abs().max()) < 2 ** 13 and torch.equal(z * 1024, (z * 1024).round())
        top2 = z.topk(2, dim=1).values
        assert bool((top2[:, 0] > top2[:, 1]).all())
        zero = x.sum(1) == 0
        assert int(zero.sum()) >= B // 8 and bool((z[zero] < 0).all())
        assert bool((z.argmax(1)[zero] == fx.y.long()[zero]).all())


SAT_GUARDS = [(32, 4, "bf16", o, 0) for o in ("sgd", "adam")] + [(512, 3, "bf16", o, 0) for o in ("sgd", "adam")] + \
             [(512, 3, "fp8", "adam", 7), (128, 4, "fp8", "sgd", 0)]


@pytest.mark.parametrize("B,S,dtype,opt,base", SAT_GUARDS)
def test_sat_fixture_guards(B, S, dtype, opt, base):
    fx = sat_fixture(B, S, seed=B + S)
    margins = sat_guard(fx, dtype == "fp8", opt, base)
    assert min(margins) >= 112


# ------------------------------------------------------------------------------ GPU runs
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def expected_bm_w(D, H):
    """The launcher's weight-gradient tile height: 64 rows unless dW1's tiles + dW2's + the bias CTA
    would exceed one CTA per SM."""
    nt_d, nt_h = -(-D // 64), -(-H // 64)
    return 64 if -(-H // 64) * nt_d + nt_h + 1 <= sms() else 128


def allowed_plans(plan, D, H, C, B):
    """Plans the launcher may run for a request: 3 and 4 need hidden 256 and 57..64 classes, else
    plan 0; plan 4 becomes 3 where the grid rounded up to whole 4-CTA clusters exceeds the SM count,
    or where cudaOccupancyMaxActiveClusters reports fewer clusters than the grid needs.  That count
    is not visible from Python, so this assumes it: the device holds at least 16 clusters of four
    at once (a grid of up to 64 CTAs, B = 1024; an H100 with 132 SMs does, and
    test_gpu_mlp_chain64.py relies on the same).  Between 64 CTAs and the SM count (B = 2048) either
    plan is accepted, and the case prints which one ran."""
    ncp = (C + 7) // 8 * 8
    if plan == 0 or H != 256 or ncp != 64:
        return {0}
    if plan == 3:
        return {3}
    nt_d = -(-D // 64)
    bm_w = expected_bm_w(D, H)
    grid = max(-(-B // 64) * 4, -(-H // bm_w) * nt_d + 4 + 1, 32)
    grid4 = -(-grid // 4) * 4
    if grid4 > sms():
        return {3}
    return {4} if grid4 <= 64 else {3, 4}


def ran_plan(d):
    """Phase plan and optimizer placement from CTA 0's stamps of step row d: slot 6 (whole h tile
    landed) exists only in the chain plans, and plan 4 hands its h slice over (slot 1) before its
    fwd1 epilogue ends (slot 17) while plans 0 and 3 stamp slot 1 after the grid barrier that
    follows it; slot 5 (after the flat optimizer phase) exists only with epiopt = 0."""
    assert int(d[17]) > 0 and int(d[1]) > 0
    chain = int(d[6]) > 0
    plan = (4 if int(d[1]) <= int(d[17]) else 3) if chain else 0
    return plan, 0 if int(d[5]) > 0 else 1


class Run:
    """A FlatMLP over a fixture's parameters and inputs on the GPU, with what the launch read
    snapshotted before it runs."""

    def __init__(self, fx, fp8, opt, base=None, moments_seed=None):
        from bflc_demo_b200._native import C
        self.fx, self.fp8, self.opt = fx, fp8, opt
        self.B = fx.B
        self.spec = mlp_spec(fx.D, fx.H, fx.C)
        dev = "cuda"
        rows = fx.xu8.shape[0]
        xu8 = fx.xu8.to(dev)
        self.xb = torch.empty(rows, fx.D, device=dev, dtype=BF16)
        xq = torch.zeros(rows, fx.D, device=dev, dtype=torch.uint8)
        xsf = torch.full((sf_bytes(rows, fx.D),), 127, device=dev, dtype=torch.uint8)
        self.x_dq = torch.empty(rows, fx.D, device=dev, dtype=BF16)
        C().prep_inputs(xu8, self.xb, xq, xsf, 1.0 / 255.0, self.x_dq)
        self.y = fx.y.to(dev)
        master = fx.master.to(dev).clone()
        self.step = torch.full((1,), base or 0, device=dev, dtype=torch.int32)
        self.tr = FlatMLP(self.spec, master, master.bfloat16(), torch.zeros_like(master), self.B,
                          optimizer=opt, lr=LR[opt], fp8=fp8,
                          step_dev_ptr=self.step.data_ptr() if base is not None else 0)
        if opt == "adam" and moments_seed is not None:
            g = torch.Generator().manual_seed(moments_seed)
            self.tr.m.copy_(torch.randn(self.spec.total, generator=g) * 1e-3)
            self.tr.v.copy_(torch.rand(self.spec.total, generator=g) * 1e-6)
        if fp8:
            self.tr.quantize_weights()
        self.bar = torch.zeros(1, device=dev, dtype=torch.int32)
        self.dbg = None

    def launch(self, plan, epiopt, steps, row0=0):
        tr = self.tr
        rows = slice(row0, row0 + steps * self.B)
        self.bar.zero_()
        self.dbg = torch.zeros(steps, 32, device="cuda", dtype=torch.int64)
        tr.train_epoch_fused(self.xb[rows], self.y[rows], steps, self.bar.data_ptr(), self.dbg, plan, epiopt,
                             **({"x_dq": self.x_dq[rows]} if self.fp8 else {}))
        torch.cuda.synchronize()

    def state(self):
        tr = self.tr
        out = {"master": tr.master.clone(), "shadow": tr.shadow.clone(), "grad": tr.grad.clone(),
               "h": tr.h.clone(), "dlogits": tr.dlogits.clone(), "dh": tr.dh.clone(),
               "loss": float(tr.loss_sum), "correct": int(tr.correct)}
        if self.opt == "adam":
            out["m"], out["v"] = tr.m.clone(), tr.v.clone()
        if self.fp8:
            out["work_q"], out["work_dq"], out["h_dq"] = tr.work_q.clone(), tr.work_dq.clone(), tr.h_dq.clone()
        return out


def mx8_ambiguous(h):
    """Elements of a bf16 h [R, 256] whose e4m3 quantisation may differ between the fp32 value the
    kernel quantises and its bf16 rounding: h exactly on an e4m3 midpoint at the group's scale, or
    any element of a group whose amax / 448 is a power of two (the scale byte's threshold: the
    fp32 amax may take the next scale, whose grid is twice as coarse).  Elsewhere round-to-nearest
    keeps the fp32 value and its bf16 rounding on the same side of every decision.  Returns the
    mask, how far the two dequantised candidates can lie apart, and where one of them may be 0."""
    R, K = h.shape
    hd = h.double().view(R, K // 32, 32)
    amax = hd.abs().amax(-1, keepdim=True)
    mant, _ = torch.frexp(amax / 448)
    grp = ((amax > 0) & (mant == 0.5)).expand_as(hd)
    e = torch.where(amax > 0, torch.ceil(torch.log2(amax / 448)).clamp(-124, 127), torch.zeros_like(amax))
    s = (hd * torch.exp2(-e)).abs()
    spacing = torch.where(s >= 2.0 ** -6, torch.exp2(torch.floor(torch.log2(s.clamp_min(2.0 ** -6))) - 3),
                          torch.full_like(s, 2.0 ** -9))
    q = s / (spacing / 2)
    mid = (q == q.round()) & (q.round() % 2 == 1)
    amb = mid | grp
    step = torch.where(grp, 2 * spacing, spacing) * torch.exp2(e) * amb
    may_zero = amb & (s <= 2.0 ** -8)
    return amb.view(R, K), step.view(R, K), may_zero.view(R, K)


def check_one_step(fx, fp8, plan, epiopt, opt, base=None):
    """One single-step launch, every stage against fp64 from the kernel's own upstream intermediates."""
    run = Run(fx, fp8, opt, base=base, moments_seed=(17 if base else None))
    tr, spec, B, C, D, H = run.tr, run.spec, fx.B, fx.C, fx.D, fx.H
    p0 = {k: t.double() for k, t in spec.views(tr.master.clone()).items()}
    s0 = {k: t.double() for k, t in spec.views(tr.shadow.clone()).items()}
    m0 = tr.m.double().clone() if opt == "adam" else None
    v0 = tr.v.double().clone() if opt == "adam" else None
    wdq0 = tr.work_dq.double().clone() if fp8 else None
    run.launch(plan, epiopt, 1)
    out = run.state()

    got_plan, got_eo = ran_plan(run.dbg.cpu()[0])
    assert got_plan in allowed_plans(plan, D, H, C, B), (plan, got_plan)
    assert got_eo == epiopt
    info = f"plan {got_plan}, epiopt {got_eo}, bm_w {expected_bm_w(D, H)} on {sms()} SMs"

    x = run.xb[:B].double()
    xf = run.x_dq[:B].double() if fp8 else x
    if fp8:
        w1f = wdq0[:H * D].view(H, D)
        w2f = wdq0[H * D:H * D + 64 * H].view(64, H)[:C]
    else:
        w1f, w2f = s0["w1"], s0["w2"]
    w2s = s0["w2"]

    # ---- h = bf16(relu(x W1^T + b1))
    h_ref = torch.relu(xf @ w1f.t() + p0["b1"])
    if fx.kind == "int":
        assert_exact(out["h"], h_ref, f"h ({info})")
    else:
        assert_bound(out["h"], h_ref, gamma(D + 1) * (xf.abs() @ w1f.abs().t() + p0["b1"].abs()) * (1 + 2.0 ** -7),
                     f"h ({info})")
    h = out["h"].double()
    # fp8: fwd2 reads h quantised to MXFP8 (h_dq).  Plan 3 stores it and reloads it by TMA; plan 4
    # hands it over on chip and leaves the global h_dq unwritten, so there fwd2's operand is the
    # quantiser's output, up to the elements mx8_ambiguous names.
    hstep = torch.zeros_like(h)
    may_zero = torch.zeros_like(h, dtype=torch.bool)
    if fp8:
        want = quantize_mx8_reference(out["h"].float()).dequantize().to(BF16)
        if fx.kind == "real":
            amb, hstep, may_zero = mx8_ambiguous(out["h"])
        else:
            amb = torch.zeros_like(may_zero)
        if got_plan == 3:
            bad = out["h_dq"].view(torch.int16) != want.view(torch.int16)
            assert not bool((bad & ~amb).any()), f"h_dq: {int((bad & ~amb).sum())} elements off the quantiser ({info})"
            hin = out["h_dq"].double()
            hstep.zero_()
            may_zero.zero_()
        else:
            hin = want.double()
    else:
        hin = h

    # ---- logits (fp64 from the kernel's h / h_dq), dlogits, loss, correct
    y = run.y[:B]
    z = hin @ w2f.t() + p0["b2"]
    ez = gamma(H + 1) * ((hin.abs() + hstep) @ w2f.abs().t() + p0["b2"].abs()) + hstep @ w2f.abs().t()
    _, dl_ref, loss_ref = softmax_xent(z, y, B)
    sdl = softmax_slack(z, ez, y, B)
    dl = out["dlogits"]
    assert_bound(dl[:, :C], dl_ref, sdl * (1 + 2.0 ** -7), f"dlogits ({info})")
    assert int(torch.count_nonzero(dl[:, C:])) == 0, "padded dlogits columns"
    top2 = z.topk(2, dim=1)
    hits = top2.indices[:, 0] == y.long()
    if fx.kind == "int":
        assert bool((top2.values[:, 0] > top2.values[:, 1]).all())
        assert out["correct"] == int(hits.sum()), (out["correct"], int(hits.sum()), info)
    else:
        sure = top2.values[:, 0] - top2.values[:, 1] > 2 * ez.amax(1)
        lo, und = int((hits & sure).sum()), int((~sure).sum())
        assert lo <= out["correct"] <= lo + und, (out["correct"], lo, und, info)
        if not bool(hstep.any()):   # plan 4 fp8: the ambiguous h_dq elements leave more rows open
            assert und <= max(2, B // 20), und
    zmax = z.amax(1)
    t = (z - zmax[:, None]).abs() + 2 * ez.amax(1, keepdim=True)
    r_sum = (U * t + (2 + 1.173 * t) * ULP).amax(1) + gamma(C)
    lse = torch.logsumexp(z, 1)
    row_err = (2 * ez.amax(1) + r_sum * (1 + 2 * r_sum) + 3 * 2.0 ** -21
               + 2 * U * ((lse - zmax).abs() + zmax.abs() + loss_ref.abs()))
    loss_slack = float(row_err.sum()) + gamma(B + 32) * float(loss_ref.abs().sum())
    assert abs(out["loss"] - float(loss_ref.sum())) <= loss_slack, (out["loss"], float(loss_ref.sum()), info)

    # ---- dh = (dlogits W2) * mask (mask: h > 0, fp8: h_dq > 0), from the kernel's dlogits
    dlk = dl[:, :C].double()
    mask = (hin > 0).double()
    a = dlk @ w2s
    sa = gamma(C) * (dlk.abs() @ w2s.abs()) * mask + a.abs() * may_zero
    assert_bound(out["dh"], a * mask, sa * (1 + 2.0 ** -7), f"dh ({info})")

    # ---- gradients (from the kernel's dh, dlogits, bf16 h and x) and the update
    dhk = out["dh"].double()
    g = {"w1": dhk.t() @ x, "w2": dlk.t() @ h, "b1": (a * mask).sum(0), "b2": dl_ref.sum(0)}
    sg = {"w1": gamma(B) * (dhk.abs().t() @ x.abs()), "w2": gamma(B) * (dlk.abs().t() @ h.abs()),
          "b1": sa.sum(0) * (1 + gamma(B)) + gamma(B) * (a * mask).abs().sum(0),
          "b2": sdl.sum(0) * (1 + gamma(B)) + gamma(B) * dl_ref.abs().sum(0)}
    pm = spec.views(out["master"])
    lr = f32(LR[opt])
    if opt == "sgd":
        for k in ("w1", "b1", "w2", "b2"):
            want = sgd(p0[k], g[k], lr)
            slack = lr * sg[k] * (1 + 2 * U) + 2 * U * lr * (g[k].abs() + sg[k])
            assert_bound(pm[k], want, slack, f"SGD {k} ({info})")
    else:
        tt = (base or 0) + 1
        mv0 = {k: t for k, t in spec.views(m0).items()}
        vv0 = {k: t for k, t in spec.views(v0).items()}
        mm, vm = spec.views(out["m"]), spec.views(out["v"])
        for k in ("w1", "b1", "w2", "b2"):
            (w, m, v), (sw, sm, sv) = adam_slack(p0[k], mv0[k], vv0[k], g[k], sg[k], lr, tt)
            assert_bound(mm[k], m, sm, f"Adam m {k} ({info})")
            assert_bound(vm[k], v, sv, f"Adam v {k} ({info})")
            assert_bound(pm[k], w, sw, f"Adam w {k} (tt {tt}, {info})")
    assert torch.equal(out["shadow"], out["master"].bfloat16()), "shadow != bf16(master')"
    assert int(torch.count_nonzero(out["grad"])) == 0, "gradient buffer not re-zeroed"
    if fp8:
        tr.quantize_weights()
        torch.cuda.synchronize()
        L = tr.ql
        for name, nbytes in (("w1q", H * D), ("w1sf", -(-H // 128) * L["kb1"] * 512), ("w2q", 64 * H),
                             ("w2sf", L["kb2"] * 512)):
            sl = slice(L[name], L[name] + nbytes)
            assert torch.equal(out["work_q"][sl], tr.work_q[sl]), name
        assert torch.equal(out["work_dq"], tr.work_dq), "work_dq"
    print(f"[trainer conformance] {fx.kind} B={B} {D}-{H}-{C} {'fp8' if fp8 else 'bf16'} {opt}: {info}")
    return got_plan


# bench shape 784-256-62, B = 512: every combination the launcher accepts
BENCH = ([("bf16", p, eo, o, k) for p in (0, 3, 4) for eo in (0, 1) for o in ("sgd", "adam") for k in ("int", "real")]
         + [("fp8", p, 1, o, k) for p in (3, 4) for o in ("sgd", "adam") for k in ("int", "real")])


@gpu
@pytest.mark.parametrize("dtype,plan,epiopt,opt,kind", BENCH,
                         ids=[f"{d}-p{p}-eo{e}-{o}-{k}" for d, p, e, o, k in BENCH])
def test_one_step_bench_shape(dtype, plan, epiopt, opt, kind):
    D, H, C, B = 784, 256, 62, 512
    fx = (int_fixture if kind == "int" else real_fixture)(D, H, C, B, seed=B + D + H + C)
    # Adam: step count 0 on the integer fixture, a carried step word of 7 (and warm moments) on the other
    base = (0 if kind == "int" else 7) if opt == "adam" else None
    check_one_step(fx, dtype == "fp8", plan, epiopt, opt, base)


SHAPES = [(128, 784, 256, 62), (200, 784, 256, 62), (1024, 784, 256, 62), (2048, 784, 256, 62),
          (256, 784, 256, 64), (256, 784, 256, 10), (256, 512, 256, 62), (128, 64, 256, 62),
          (200, 784, 128, 62), (128, 784, 640, 62)]
SHAPE_CASES = ([("bf16", p, k) + s for s in SHAPES for p in (DEFAULT_PLAN, 0) for k in ("int", "real")]
               + [("fp8", DEFAULT_PLAN, k) + s for s in SHAPES for k in ("int", "real")
                  if s[0] % 128 == 0 and s[2] == 256 and 57 <= s[3] <= 64])


@gpu
@pytest.mark.parametrize("dtype,plan,kind,B,D,H,C", SHAPE_CASES,
                         ids=[f"{d}-p{p}-{k}-B{b}-{dd}x{h}x{c}" for d, p, k, b, dd, h, c in SHAPE_CASES])
def test_one_step_shapes_and_tails(dtype, plan, kind, B, D, H, C):
    """Tail rows (B = 200: 64- and 128-row tails), 16 and 32 clusters, no padded classes, ncp = 16,
    no K tail, one K-block, hidden 128 and 640 (plan 0; 128-row weight-gradient tiles on a
    132-SM part).  SGD on the integer fixture, Adam with a carried step word on the other."""
    fx = (int_fixture if kind == "int" else real_fixture)(D, H, C, B, seed=B + D + H + C)
    opt = "sgd" if kind == "int" else "adam"
    check_one_step(fx, dtype == "fp8", plan, 1, opt, 7 if opt == "adam" else None)


REJECTED = [("plan0", 0, 1, 256), ("flat-optimizer-phase", 4, 0, 256), ("B-not-multiple-of-128", 4, 1, 200)]


@gpu
@pytest.mark.parametrize("what,plan,epiopt,B", REJECTED, ids=[r[0] for r in REJECTED])
def test_fp8_rejected_combinations_raise(what, plan, epiopt, B):
    fx = real_fixture(784, 256, 62, B, seed=5)
    run = Run(fx, True, "sgd")
    before = run.tr.master.clone()
    with pytest.raises(RuntimeError):
        run.launch(plan, epiopt, 1)
    torch.cuda.synchronize()
    assert torch.equal(run.tr.master, before)


# --------------------------------------------------------- multi-step launch against replay
REPLAY = ([("bf16", p, o, B, S, 0) for p in (0, 3, 4) for o in ("sgd", "adam") for B, S in ((32, 4), (512, 3))]
          + [("fp8", 4, "adam", 512, 3, 7), ("fp8", 3, "sgd", 128, 4, 0)])


@gpu
@pytest.mark.parametrize("dtype,plan,opt,B,S,base", REPLAY,
                         ids=[f"{d}-p{p}-{o}-B{b}-S{s}-base{t}" for d, p, o, b, s, t in REPLAY])
def test_steps_in_one_launch_match_single_step_replay(dtype, plan, opt, B, S, base):
    """S steps in one launch against the same S steps as S single-step launches (Adam: step word
    base + s): the r0 row offsets into x and the labels, tt, the ring / accumulator / chain /
    barrier parities across steps, the refresh of the work copies between steps and, at B = 32,
    that rows 32..63 of the last M-tile (the next step's x) never reach an output.  The saturated
    fixture makes every float-atomic sum exact, so everything but the loss is bit-equal."""
    fp8 = dtype == "fp8"
    fx = sat_fixture(B, S, seed=B + S)
    sb = base if opt == "adam" else None
    one = Run(fx, fp8, opt, base=sb)
    one.launch(plan, 1, S)
    got = one.state()
    d = one.dbg.cpu()
    plans = {ran_plan(d[s])[0] for s in range(S)}
    assert len(plans) == 1 and plans <= allowed_plans(plan, fx.D, fx.H, fx.C, B), plans
    # saturation: dlogits of the last step are 0 or +-1/B (this also rests on __expf(0) == 1)
    dl = got["dlogits"].double()
    assert bool(((dl == 0) | (dl.abs() == 1.0 / B)).all()), "dlogits not saturated"
    rep = Run(fx, fp8, opt, base=sb)
    for s in range(S):
        if sb is not None:
            rep.step.fill_(sb + s)
        rep.launch(plan, 1, 1, row0=s * B)
    want = rep.state()
    for k in got:
        if k == "loss":
            assert abs(got[k] - want[k]) <= gamma(B * S + 32) * abs(want[k]), (got[k], want[k])
        elif k == "correct":
            assert got[k] == want[k]
        elif k == "h_dq" and plans == {4}:
            continue   # plan 4 hands h_dq over on chip and never writes the global copy
        else:
            assert torch.equal(got[k], want[k]), k
    assert int(torch.count_nonzero(got["grad"])) == 0
    print(f"[trainer replay] {dtype} plan {plans} {opt} B={B} S={S}: bit-equal")


# ------------------------------------------------------------------ the last step's upload
def _upload_round(dtype, byzantine):
    """One one-step round of a world-1 FusedEngine (SGD, so that the bias update is linear in its
    gradient): returns the engine, the genesis model and the fp32 / bf16 upload buffers and the
    fp8 blob of that round."""
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    B = 512
    cfg = FLConfig.for_world(1, model="mlp", hidden=256, batch_size=B, samples_per_client=B,
                             learning_rate=LR["sgd"], dtype=dtype, optimizer="sgd", cuda_graph=False,
                             byzantine_ranks=[0] if byzantine else [], byzantine_scale=5.0)
    eng = FusedEngine(cfg, femnist_like(1, B, seed=7, only=0)[0])
    assert eng.fused_upload and eng.steps == 1 and eng.byz == (1 if byzantine else 0)
    genesis = eng.global_master.clone()
    eng.capture()                      # one eager round: epoch 0 -> 1, uploads of parity 0
    torch.cuda.synchronize()
    assert eng.read_state()["epoch"] == 1
    o, P = eng.layout.offsets, eng.n_params
    up = eng.heap.view(o["upload_master0"], [P], torch.float32).clone()
    sh = eng.heap.view(o["upload_shadow0"], [P], torch.bfloat16).clone()
    blob = eng.heap.view(eng.upq_off[0], [eng.blob_bytes], torch.uint8).clone() if eng.fp8 else None
    return eng, genesis, up, sh, blob


def _check_upload_encoding(eng, up, sh, blob):
    """fp8: the blob (e4m3 weights, scale chunks, fp32 biases) and the upload shadow (the weights
    dequantised, the biases in bf16) are what the stand-alone quantiser makes of the fp32 upload;
    bf16: the upload shadow is bf16 of the fp32 upload."""
    spec = eng.spec
    vu, vs = spec.views(up), spec.views(sh)
    if not eng.fp8:
        for k in ("w1", "b1", "w2", "b2"):
            assert torch.equal(vs[k], vu[k].bfloat16()), k
        return
    tr, L = eng.trainer, eng.ql
    H, D = eng.cfg.hidden, eng.in_dim
    C = spec.by_name["w2"].shape[0]
    tr.quantize_weights(up)            # into the trainer's own work blob and work_dq
    torch.cuda.synchronize()
    for name, nbytes in (("w1q", H * D), ("w1sf", -(-H // 128) * L["kb1"] * 512), ("w2q", 64 * H),
                         ("w2sf", L["kb2"] * 512)):
        sl = slice(L[name], L[name] + nbytes)
        assert torch.equal(blob[sl], tr.work_q[sl]), name
    assert torch.equal(vs["w1"], tr.work_dq[:H * D].view(H, D)), "upload shadow w1"
    assert torch.equal(vs["w2"], tr.work_dq[H * D:H * D + 64 * H].view(64, H)[:C]), "upload shadow w2"
    assert torch.equal(blob[L["b1"]:L["b1"] + 4 * H].view(torch.float32), vu["b1"])
    assert torch.equal(blob[L["b2"]:L["b2"] + 4 * C].view(torch.float32), vu["b2"])
    for k in ("b1", "b2"):
        assert torch.equal(vs[k], vu[k].bfloat16()), k


@gpu
@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_last_step_publishes_the_byzantine_upload(dtype):
    """The last step's optimizer epilogue is UploadLocalUpdate; a Byzantine rank uploads
    g0 - s (w - g0) instead of w (g0 = the global model it trained from, s = byzantine_scale).  One
    one-step round on an honest and on a Byzantine engine from the same genesis and data: the
    weight matrices are bit-reproducible (no float atomic reaches them in one step), so the
    Byzantine w1 / w2 are fl(g0 - 5 (w - g0)) of the honest ones bit for bit -- with or without
    the compiler contracting the product into an FMA, one rule for the whole upload.  The biases'
    gradients are column sums: every plan adds each column's fp32 partial sums of 32 batch rows
    (the same bits in both runs) by B / 32 float atomics, whose order differs between runs, so the
    two gradients lie within 2 gamma_{B/32} of the partials' magnitudes.  Those are bounded by the
    terms' magnitudes: |dlogits| (fp32, at most 2^-7 above their bf16 copy) for db2 and
    |dlogits| |W2| (1 + gamma_C) for db1."""
    eng, g0, w, sh_h, blob_h = _upload_round(dtype, False)
    _check_upload_encoding(eng, w, sh_h, blob_h)
    C = eng.spec.by_name["w2"].shape[0]
    dl = eng.trainer.dlogits[:, :C].double().abs()
    w2s = eng.spec.views(g0)["w2"].bfloat16().double().abs()
    terms = {"b1": (dl @ w2s).sum(0) * (1 + gamma(C)) * (1 + gamma(32)),
             "b2": dl.sum(0) * (1 + 2.0 ** -7) * (1 + gamma(32))}
    del eng
    eng, g0b, wb, sh_b, blob_b = _upload_round(dtype, True)
    assert torch.equal(g0, g0b)
    _check_upload_encoding(eng, wb, sh_b, blob_b)
    spec, B = eng.spec, eng.cfg.batch_size
    vg, vw, vb = spec.views(g0), spec.views(w), spec.views(wb)
    assert float((vw["w1"] - vg["w1"]).abs().max()) > 0, "the honest round did not train"
    for k in ("w1", "w2"):
        d = vw[k] - vg[k]
        unfused = vg[k] - 5.0 * d
        fused = (vg[k].double() - 5.0 * d.double()).float()
        assert torch.equal(vb[k], unfused) or torch.equal(vb[k], fused), (
            k, int((vb[k] != unfused).sum()), int((vb[k] != fused).sum()))
    lr = f32(LR["sgd"])
    for k in ("b1", "b2"):
        dg = 2 * gamma(B // 32) * terms[k]
        g0k, wk = vg[k].double(), vw[k].double()
        ref = g0k - 5 * (wk - g0k)
        slack = 5 * (lr * dg * (1 + 2 * U) + 2 * U * wk.abs()) + 2 * U * (5 * (wk - g0k).abs() + ref.abs())
        assert_bound(vb[k], ref, slack, f"Byzantine upload {k}")
