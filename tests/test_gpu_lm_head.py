"""The vocabulary-wide cross-entropy kernel (``xent_rows``, csrc/kernels/nn_kernels.cu) and the LM head
built on it (``ops.nn.lm_xent`` / ``lm_hits``) against float64.

Bounds (fast math, as built): each exp is ex2.approx of a rounded argument (2 ulp, plus one rounding
of |x - m|), the row sum runs in fp32 over V terms (gamma_V), __logf adds 2^-21.41 absolute on
[0.5, 2] and 3 ulp elsewhere, the loss subtraction rounds once.  dlogits adds the approximate
reciprocal (2 ulp), the products (u each) and the bf16 output (half an ulp).

Argmax tie rule: the lowest column among equal maxima wins (``torch.argmax`` returns the first
maximal index too), the rule of the GEMM ARGMAX_ACC epilogue.
"""
import pytest
import torch

gpu = pytest.mark.gpu
F64 = torch.float64
ULP, U = 2.0 ** -23, 2.0 ** -24
BF_U = 2.0 ** -8
NAN = float("nan")


def gamma(n):
    return n * ULP / (1 - n * ULP)


def xent_bounds(z, t, gs):
    """z fp64 [M, V] (the fp32 logits), t [M] -> (loss, lse, p, loss bound, dlogits bound)"""
    m = z.amax(-1, keepdim=True)
    lse = torch.logsumexp(z, -1)
    p = torch.exp(z - lse[:, None])
    x = (z - m).abs()
    rp = torch.exp2((U * x) / 0.69) * (1 + 2 * ULP) - 1 + 2 * U          # one exp (argument incl.)
    V = z.shape[1]
    rs = (p * rp).sum(-1) / p.sum(-1) + gamma(V)                        # relative error of the sum
    s = torch.exp(lse - m[:, 0])
    log_err = torch.where((s >= 0.5) & (s <= 2), torch.full_like(s, 2.0 ** -21.41), 3 * ULP * torch.log(s).abs())
    loss = lse - z.gather(1, t[:, None].long())[:, 0]
    lb = rs / (1 - rs) + log_err + 2 * U * (m[:, 0].abs() + lse.abs() + loss.abs()) + 1e-30
    g = (p - torch.nn.functional.one_hot(t.long(), V).to(F64)) * gs
    db = gs * p * ((1 + rp) * (1 + rs[:, None]) / (1 - rs[:, None]) * (1 + 2 * ULP) * (1 + U) ** 3 - 1) \
        + 2 * U * gs + BF_U * g.abs() + 2.0 ** -133
    return loss, g, lb, db


def run_xent(z32, V, t, gs=1.0, ldd=None, with_loss=True, with_dl=True):
    from bflc_demo_b200._native import C
    M = z32.shape[0]
    loss = torch.full((M + 8,), NAN, device="cuda") if with_loss else None
    hits = torch.zeros(1, device="cuda", dtype=torch.int32)
    dl = torch.full((M, ldd or (V + 7) // 8 * 8 + 8), NAN, device="cuda", dtype=torch.bfloat16) if with_dl else None
    C().xent_rows(z32, V, t, loss, hits, dl, gs)
    torch.cuda.synchronize()
    return loss, hits, dl


def padded_logits(M, V, seed, scale=3.0):
    """fp32 [M, V] view of a NaN-filled [M, ld] buffer, ld > V (canaries in the pitch)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ld = (V + 3) // 4 * 4 + 4
    buf = torch.full((M, ld), NAN, device="cuda")
    buf[:, :V] = torch.randn(M, V, device="cuda", generator=g) * scale
    return buf[:, :V]


@gpu
@pytest.mark.parametrize("M", [1, 77, 130])
@pytest.mark.parametrize("V", [1000, 8192, 30522, 50257])
def test_xent_rows_matches_fp64(V, M):
    z = padded_logits(M, V, seed=V + M)
    t = torch.randint(0, V, (M,), device="cuda", dtype=torch.int32)
    gs = 1.0 / M
    loss, hits, dl = run_xent(z, V, t, gs)
    assert torch.isnan(loss[M:]).all(), "loss written past M"
    zr = z.double().cpu()
    ref_loss, ref_g, lb, db = xent_bounds(zr, t.cpu(), gs)
    err = (loss[:M].double().cpu() - ref_loss).abs()
    assert torch.isfinite(loss[:M]).all() and (err <= lb).all(), f"loss: max err {err.max()} vs bound {lb.min()}"
    d = dl.double().cpu()
    assert (d[:, V:] == 0).all(), "dlogits pad columns must be zero"
    derr = (d[:, :V] - ref_g).abs()
    assert torch.isfinite(d).all() and (derr <= db).all(), f"dlogits: {int((derr > db).sum())} elements out of bound"
    assert int(hits) == int((zr.argmax(-1) == t.cpu().long()).sum())


@gpu
def test_dominant_logit_and_ties_are_exact():
    M, V = 6, 1000
    z = torch.zeros(M, V, device="cuda")
    t = torch.tensor([5, 17, 3, 999, 40, 41], device="cuda", dtype=torch.int32)
    z[0, 5] = 200.0                       # target dominates: loss 0, dlogits 0
    z[1, 900] = 200.0                     # another column dominates: loss 200, dl = +gs at 900, -gs at 17
    z[2, 3] = z[2, 700] = 200.0           # tie, the target is the first maximum: a hit
    z[3, 2] = z[3, 999] = 200.0           # tie, the target is the second maximum: no hit
    z[4, 40] = 200.0
    z[5, 40] = z[5, 41] = 200.0           # tie, the target is the second maximum: no hit
    gs = 0.25
    loss, hits, dl = run_xent(z, V, t, gs)
    assert loss[0] == 0 and loss[1] == 200 and loss[4] == 0
    assert int(hits) == 3                 # rows 0, 2, 4
    d = dl.float()
    assert torch.count_nonzero(d[0]) == 0 and torch.count_nonzero(d[4]) == 0
    want = torch.zeros(V, device="cuda")
    want[900], want[17] = gs, -gs
    assert torch.equal(d[1, :V], want)


@gpu
def test_hits_only_mode_reads_and_writes_nothing_else():
    M, V = 300, 8192
    z = padded_logits(M, V, seed=1)
    before = z.clone()
    t = torch.randint(0, V, (M,), device="cuda", dtype=torch.int32)
    t[:50] = z[:50].argmax(-1).int()
    _, hits, _ = run_xent(z, V, t, with_loss=False, with_dl=False)
    assert int(hits) == int((z.argmax(-1) == t.long()).sum()) >= 50
    assert torch.equal(z.nan_to_num(7.0), before.nan_to_num(7.0))
    loss, hits2, dl = run_xent(z, V, t)
    assert int(hits2) == int(hits)


@gpu
@pytest.mark.parametrize("V,M", [(8192, 256), (1003, 77)])
def test_lm_xent_matches_fp64_autograd_with_tied_accumulation(V, M):
    from bflc_demo_b200.ops import nn as F
    K = 256
    g = torch.Generator(device="cuda").manual_seed(V)
    h = (torch.randn(M, K, device="cuda", generator=g)).to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(V, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    g0 = torch.randn(V, K, device="cuda", generator=g)
    gw = g0.clone()
    t = torch.randint(0, V, (M,), device="cuda", dtype=torch.int32)
    cnt = torch.zeros(1, device="cuda", dtype=torch.int32)
    prev = F.set_precision("mx8")         # the head GEMM stays bf16 regardless
    try:
        loss = F.lm_xent(h, w, gw, t, cnt)
        (loss * 0.5).backward()
    finally:
        F.set_precision(prev)
    hr = h.detach().double().cpu().requires_grad_(True)
    wr = w.double().cpu().requires_grad_(True)
    zr = hr @ wr.T
    lr = torch.nn.functional.cross_entropy(zr, t.cpu().long())
    (lr * 0.5).backward()
    # the logits: fp32 sums of K exact bf16 products; dlogits then round to bf16 (2^-8 relative)
    ez = gamma(K) * (hr.detach().abs() @ wr.detach().abs().T)
    assert abs(float(loss) - float(lr)) <= 2 * float(ez.amax(-1).mean()) + 1e-5 * abs(float(lr)) + 1e-6
    p = torch.softmax(zr.detach(), -1)
    onehot = torch.nn.functional.one_hot(t.cpu().long(), V).to(F64)
    e_dl = 0.5 / M * (p * (torch.exp(2 * ez.amax(-1, keepdim=True)) - 1) + 2 * BF_U * (p + onehot) + 1e-7)
    dh_b = e_dl @ wr.detach().abs() + gamma(V) * ((p.abs() + 1) * 0.5 / M) @ wr.detach().abs()
    assert ((h.grad.double().cpu() - hr.grad).abs() <= dh_b + BF_U * hr.grad.abs()).all()
    dgw = (gw - g0).double().cpu()
    gw_b = e_dl.T @ hr.detach().abs() + gamma(M) * (((p.abs() + 1) * 0.5 / M).T @ hr.detach().abs()) \
        + U * g0.abs().double().cpu() * 2
    assert ((dgw - wr.grad).abs() <= gw_b).all()
    assert 0 <= int(cnt) <= M


@gpu
def test_lm_hits_chunks_agree():
    from bflc_demo_b200.ops import nn as F
    M, K, V = 1000, 128, 8192
    g = torch.Generator(device="cuda").manual_seed(2)
    h = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(V, K, device="cuda", generator=g).to(torch.bfloat16)
    t = torch.randint(0, V, (M,), device="cuda", dtype=torch.int32)
    z = (h.float() @ w.float().T)
    t[::3] = z[::3].argmax(-1).int()
    counts = []
    for rows in (M, 256, 77):
        c = torch.zeros(1, device="cuda", dtype=torch.int32)
        F.lm_hits(h, w, t, c, rows)
        counts.append(int(c))
    assert counts[0] == counts[1] == counts[2] >= M // 3 - 5
