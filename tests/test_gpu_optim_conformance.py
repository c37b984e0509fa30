"""Conformance of the flat optimizer kernels (``csrc/kernels/elementwise_optim.cu``) against the exact
specification in ``test_optim_spec_host.py``, element by element.

* ``optim_step`` (SGD, Adam) and ``optim_recipe_step`` (SGD, Adam): SGD weights, Adam moments, the
  bf16 shadow (round to nearest even of the kernel's own new weight) and the cleared gradient bit for
  bit; Adam weights within the derived bound of the last line.  n covers the float4 body, the scalar
  tail and more than one grid-stride pass (1,081,357 > 132 * 8 CTAs * 256 threads * 4 floats);
  values include signed zeros, flushed subnormals, gradients whose square underflows (v -> 0) or
  overflows (v -> inf), NaN / inf gradients (plain path: they propagate) and bf16 ties.
* Recipe: every schedule with s below, at and above the warmup and at and above the total; random
  no-decay masks (the tail's block and bit 31 of a word set); decay 0 and 0.1; the clip coefficient
  from a real ``grad_norm`` launch (triggered and not) and from a header written here (0.375); the
  skipped step; the device predicate.
* ``grad_norm``: norm, coefficient, non-finite flag, skip counter, ticket reset and predicate.
* ``cast_f32_to_bf16``, ``cast_u8_to_bf16``, ``add_bf16``: every rounding class over every tail length.
* ``FlatMLP.optimizer_step`` (Adam, a device step word): the arguments the model passes.
* The bindings refuse short, misaligned, strided or mistyped buffers and an Adam step below 1.  Every
  refused buffer goes either to a predicated entry point with the predicate word 0 (the kernel would
  return before touching memory) or stays in bounds and aligned, so no refusal test could fault the
  device if its check were missing.

Every output buffer extends past n with NaN canaries that must survive bit for bit.
"""
import numpy as np
import pytest
import torch

from test_optim_spec_host import (F32, N_OPT, SH_INIT, BF16_TIES, Case, add_bf16_spec, bits32, cast_u8_spec,
                                  check_update, clip_spec, first_bad, grad_norm_spec, plain_cases, recipe_cases,
                                  rne_bf16, run_update, same_bf16, same_bits, values)

pytestmark = pytest.mark.gpu

PAD = 64
CAN32 = 0x7FC00ABC         # fp32 NaN canary past n
CAN16 = 0x7FC3             # bf16 NaN canary past n


def C():
    from bflc_demo_b200._native import C as _C
    return _C()


def f32_buf(x):
    n = len(x)
    a = np.empty(n + PAD, F32)
    a[:n] = x
    a.view(np.uint32)[n:] = CAN32
    return torch.from_numpy(a).cuda()


def bf16_buf(n, init=None):
    a = np.full(n + PAD, CAN16, np.uint16)
    a[:n] = SH_INIT if init is None else init
    return torch.from_numpy(a.view(np.int16)).cuda().view(torch.bfloat16)


def f32_out(buf, n, name, bad):
    a = buf.cpu().numpy()
    if not (a.view(np.uint32)[n:] == CAN32).all():
        bad.append(f"{name}: canary past n overwritten")
    return a[:n].copy()


def bf16_out(buf, n, name, bad):
    a = buf.view(torch.int16).cpu().numpy().view(np.uint16)
    if not (a[n:] == CAN16).all():
        bad.append(f"{name}: canary past n overwritten")
    return a[:n].copy()


def _ws(coef=None, nonfinite=0):
    ws = torch.zeros(C().grad_norm_workspace_bytes(), dtype=torch.uint8, device="cuda")
    if coef is not None:
        hdr = np.array([F32(coef)], F32).view(np.uint8).tolist() + np.array([nonfinite], np.int32).view(np.uint8).tolist()
        ws[:8] = torch.tensor(hdr, dtype=torch.uint8)
    return ws


def launch(c: Case, active=None, ws=None):
    """Run case c through optim_step / optim_recipe_step on canaried buffers; the outputs as numpy."""
    n, bad = c.n, []
    W, G = f32_buf(c.w), f32_buf(c.g)
    M, V = (f32_buf(c.m), f32_buf(c.v)) if c.adam else (None, None)
    SH = bf16_buf(n)
    word = torch.tensor([c.word], dtype=torch.int32, device="cuda") if c.word is not None else None
    wp = word.data_ptr() if word is not None else 0
    ap = active.data_ptr() if active is not None else 0
    mv = (M[:n], V[:n]) if c.adam else (None, None)
    if c.recipe:
        if ws is None and c.clip == "header":
            ws = _ws(c.coef, c.nonfinite)
        mask = torch.from_numpy(c.mask).cuda() if c.mask is not None else None
        C().optim_recipe_step(c.adam, W[:n], G[:n], SH[:n], *mv, c.lr, c.b1, c.b2, c.eps, c.step, wp, c.decay, mask,
                              c.schedule, c.W, c.T, ws if c.clip else None, active_ptr=ap, zero_grad=c.zero_grad)
    else:
        C().optim_step(c.adam, W[:n], G[:n], SH[:n], *mv, c.lr, c.wd, c.b1, c.b2, c.eps, c.step, wp, ap,
                       c.zero_grad)
    torch.cuda.synchronize()
    out = {"w": f32_out(W, n, "w", bad), "grad": f32_out(G, n, "grad", bad), "shadow": bf16_out(SH, n, "shadow", bad)}
    if c.adam:
        out["m"], out["v"] = f32_out(M, n, "m", bad), f32_out(V, n, "v", bad)
    else:
        out["m"], out["v"] = c.m, c.v
    return out, [f"{c.label} {b}" for b in bad]


def assert_conforms(c, out, bad):
    bad = bad + check_update(c, out)
    assert not bad, "\n".join(bad[:12])


# ------------------------------------------------------------------------------ plain optim_step
@pytest.mark.parametrize("n", N_OPT)
@pytest.mark.parametrize("adam", [False, True], ids=["sgd", "adam"])
def test_plain_step(adam, n):
    for c in plain_cases(adam, n):
        assert_conforms(c, *launch(c))


@pytest.mark.parametrize("adam", [False, True], ids=["sgd", "adam"])
def test_plain_step_predicate_off_changes_nothing(adam):
    c = plain_cases(adam, 4099)[2]
    off = torch.zeros(1, dtype=torch.int32, device="cuda")
    out, bad = launch(c, active=off)
    for k in ("w", "grad", "m", "v"):
        ok = same_bits(out[k], getattr(c, {"grad": "g"}.get(k, k)))
        bad += [] if ok.all() else [f"{k} changed at {first_bad(ok)}"]
    bad += [] if (out["shadow"] == SH_INIT).all() else ["shadow written"]
    assert not bad, bad


# ------------------------------------------------------------------------------ recipe
@pytest.mark.parametrize("n", N_OPT)
@pytest.mark.parametrize("adam", [False, True], ids=["sgd", "adam"])
def test_recipe_step(adam, n):
    for c in recipe_cases(adam, n):
        out, bad = launch(c)
        sp = run_update(c)
        if float(sp["lr"]) == 0 and c.decay == 0:
            # lr_t = 0 leaves normal weights bit-unchanged (a zero may change sign: -0 + +0 = +0)
            normal = np.abs(c.w) >= 2.0 ** -126
            ok = same_bits(out["w"], c.w) | ~normal
            bad += [] if ok.all() else [f"{c.label}: lr_t = 0 moved w at {first_bad(ok)}"]
        assert_conforms(c, out, bad)


@pytest.mark.parametrize("n", [3, 257, 4099, 100004, 1081344 + 13])
@pytest.mark.parametrize("adam", [False, True], ids=["sgd", "adam"])
def test_recipe_step_with_grad_norm_coefficient(adam, n):
    """The clip coefficient as grad_norm writes it (triggered: c = norm / 2; untriggered: c = 3e38),
    checked exactly, then consumed by the update as its PDL successor."""
    for j, trig in enumerate((True, False)):
        cs = recipe_cases(adam, n)
        c = cs[(4 * j + 1) % len(cs)]
        c.g = np.where(c.g == 0, F32(0.25), c.g).astype(F32)      # small n: all edges, g = 0 -> norm 0
        norm_ref, amb = grad_norm_spec(c.g)
        cmax = float(norm_ref) * 0.5 if trig else 3e38
        ws, norms = _ws(), torch.full((1,), -1.0, device="cuda")
        G = f32_buf(c.g)
        C().grad_norm(G[:n], ws, norms, 0, cmax)
        torch.cuda.synchronize()
        nk = F32(norms.item())
        assert same_bits(nk, norm_ref) or (amb and abs(int(bits32(nk)) - int(bits32(norm_ref))) <= 1), (nk, norm_ref)
        hdr = ws[:12].cpu().numpy()
        coef, bad_flag = hdr[:4].view(F32)[0], int(hdr[4:8].view(np.int32)[0])
        assert (coef, bad_flag) == clip_spec(nk, cmax) and (coef < 1) == trig
        c.clip, c.coef, c.label = "norm", float(coef), c.label + f" norm-clip trig={trig}"
        assert_conforms(c, *launch(c, ws=ws))


@pytest.mark.parametrize("zero_grad", [True, False])
@pytest.mark.parametrize("adam", [False, True], ids=["sgd", "adam"])
def test_recipe_skipped_step(adam, zero_grad):
    for n in (5, 4099):
        c = recipe_cases(adam, n)[2]
        c.clip, c.nonfinite, c.zero_grad, c.label = "header", 1, zero_grad, c.label + " skipped"
        assert_conforms(c, *launch(c))


@pytest.mark.parametrize("adam", [False, True], ids=["sgd", "adam"])
def test_recipe_predicate_off_changes_nothing(adam):
    c = recipe_cases(adam, 4099)[0]
    out, bad = launch(c, active=torch.zeros(1, dtype=torch.int32, device="cuda"))
    for k in ("w", "grad", "m", "v"):
        ok = same_bits(out[k], getattr(c, {"grad": "g"}.get(k, k)))
        bad += [] if ok.all() else [f"{k} changed at {first_bad(ok)}"]
    bad += [] if (out["shadow"] == SH_INIT).all() else ["shadow written"]
    assert not bad, bad


# ------------------------------------------------------------------------------ gradient norm
def _norm_grad(n, kind):
    rng = np.random.default_rng(n + len(kind))
    g = (rng.standard_normal(n) * 1e-2).astype(F32)
    if kind == "subnormal":               # only subnormals: 0 when flushed, >= 2^-126 (n >= 2) if not
        g = np.where(rng.random(n) < 0.5, 1, -1).astype(F32) * np.uint32(0x007FFFFF).view(F32)
    elif kind == "mixed":
        g[::7] = 1e-40
        g[1::11] = 3e5
    elif kind == "nan":
        g[n // 2] = np.nan
    elif kind == "inf":
        g[-1] = -np.inf
    elif kind == "overflow":              # finite, but the norm overflows fp32 (n >= 2)
        g[:] = 3e38
    return g


@pytest.mark.parametrize("kind", ["random", "mixed", "subnormal", "nan", "inf", "overflow"])
@pytest.mark.parametrize("n", N_OPT)
def test_grad_norm(n, kind):
    g = _norm_grad(n, kind)
    ref, amb = grad_norm_spec(g)
    G, ws = f32_buf(g), _ws()
    norms = torch.full((2,), -1.0, device="cuda")
    skipped = torch.full((1,), 5, dtype=torch.int32, device="cuda")
    off = torch.zeros(1, dtype=torch.int32, device="cuda")
    C().grad_norm(G[:n], ws, norms, 1, 0.75, skipped, off.data_ptr())        # predicate off: nothing
    torch.cuda.synchronize()
    assert norms.tolist() == [-1.0, -1.0] and int(skipped) == 5 and int(ws.count_nonzero()) == 0
    for rep in range(2):                                                    # the ticket resets itself
        C().grad_norm(G[:n], ws, norms, 1, 0.75, skipped)
        torch.cuda.synchronize()
        bad = []
        gk = f32_out(G, n, "grad", bad)
        assert not bad and same_bits(gk, g).all()
        nk = F32(norms[1].item())
        assert float(norms[0]) == -1.0
        assert same_bits(nk, ref) or (amb and abs(int(bits32(nk)) - int(bits32(ref))) <= 1), (nk, ref, amb)
        hdr = ws[:16].cpu().numpy()
        coef, flag, ticket = hdr[:4].view(F32)[0], int(hdr[4:8].view(np.int32)[0]), int(hdr[8:12].view(np.uint32)[0])
        assert (coef, flag) == clip_spec(nk, 0.75) and ticket == 0
        assert flag == int(kind in ("nan", "inf") or (kind == "overflow" and n >= 2))
        assert int(skipped) == 5 + (rep + 1) * flag


# ------------------------------------------------------------------------------ casts and add
def _cast_inputs(n, seed):
    rng = np.random.default_rng(seed)
    x = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    hi = rng.integers(0, 2 ** 16, 64, dtype=np.uint64).astype(np.uint32) << 16
    special = np.concatenate([
        hi | 0x8000, hi | 0x7FFF, hi | 0x8001, hi | 0x0001,                  # ties both ways, +-1 around them
        rng.integers(1, 2 ** 23, 32, dtype=np.uint64).astype(np.uint32),      # subnormals
        np.array(BF16_TIES + [0x7F7FFFFF, 0xFF7FFFFF, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFA00001,
                              0x00000000, 0x80000000, 0x007FFFFF, 0x807F8000], np.uint32)])
    k = min(len(special), n)
    x[:k] = special[:k]
    if n >= 2 * k:
        x[n - k:] = special[:k]
    return x.view(F32)


@pytest.mark.parametrize("n", [8 * 40 + r for r in range(8)] + [1, 7, 100003])
def test_cast_f32_to_bf16(n):
    x = _cast_inputs(n, n)
    X, D, bad = f32_buf(x), bf16_buf(n), []
    C().cast_f32_to_bf16(X[:n], D[:n])
    torch.cuda.synchronize()
    d = bf16_out(D, n, "dst", bad)
    ok = same_bf16(d, rne_bf16(x))
    assert not bad and ok.all(), (bad, first_bad(ok))


@pytest.mark.parametrize("r", range(16))
def test_cast_u8_to_bf16(r):
    n = 512 + r
    rng = np.random.default_rng(r)
    u = rng.permutation(np.concatenate([np.arange(256), rng.integers(0, 256, n - 256)]).astype(np.uint8))
    src = torch.from_numpy(np.concatenate([u, np.full(PAD, 0xAB, np.uint8)])).cuda()
    for scale in (1 / 255.0, 1.0, 0.5, 2.0 ** -10, 3e-3):
        D, bad = bf16_buf(n), []
        C().cast_u8_to_bf16(src[:n], D[:n], scale)
        torch.cuda.synchronize()
        ok = same_bf16(bf16_out(D, n, "dst", bad), cast_u8_spec(u, scale))
        assert not bad and ok.all(), (scale, bad, first_bad(ok))
    off = torch.zeros(1, dtype=torch.int32, device="cuda")
    D = bf16_buf(n)
    C().set_predicate(off.data_ptr())
    try:
        C().cast_u8_to_bf16(src[:n], D[:n], 1.0)
    finally:
        C().set_predicate(0)
    torch.cuda.synchronize()
    assert (bf16_out(D, n, "dst", []) == SH_INIT).all()


def test_cast_u8_to_bf16_large():
    n = 100003
    u = np.random.default_rng(0).integers(0, 256, n, dtype=np.uint8)
    D, bad = bf16_buf(n), []
    C().cast_u8_to_bf16(torch.from_numpy(u).cuda(), D[:n], 1 / 255.0)
    torch.cuda.synchronize()
    assert same_bf16(bf16_out(D, n, "dst", bad), cast_u8_spec(u, 1 / 255.0)).all() and not bad


@pytest.mark.parametrize("n", [8 * 64 + r for r in range(8)] + [3])
def test_add_bf16(n):
    rng = np.random.default_rng(n)
    gap = np.arange(n) % 31                                   # exponent gaps 0 .. 30
    ea = rng.integers(40, 200, n)
    sa, sb = rng.integers(0, 2, n) << 15, rng.integers(0, 2, n) << 15
    a = (sa | (ea << 7) | rng.integers(0, 128, n)).astype(np.uint16)
    b = (sb | ((ea - gap) << 7) | rng.integers(0, 128, n)).astype(np.uint16)
    spec_pairs = [(0x7F80, 0xFF80), (0x7FC0, 0x3F80), (0x7F80, 0x3F80), (0x0001, 0x0003), (0x807F, 0x0040),
                  (0x8000, 0x8000), (0x0000, 0x8000), (0x7F7F, 0x7F7F), (0x3F80, 0x0001), (0x3F81, 0xBF80)]
    for j, (x, y) in enumerate(spec_pairs[:n]):
        a[j], b[j] = x, y
        a[n - 1 - j], b[n - 1 - j] = y, x
    A, B, O = (bf16_buf(n, init) for init in (a, b, None))
    C().add_bf16(A[:n], B[:n], O[:n])
    torch.cuda.synchronize()
    bad = []
    ok = same_bf16(bf16_out(O, n, "out", bad), add_bf16_spec(a, b))
    assert not bad and ok.all(), (bad, first_bad(ok))


# ------------------------------------------------------------------------------ production call path
def test_flat_mlp_adam_step_with_step_word():
    from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec
    spec = mlp_spec(784, 256, 62)
    n = spec.total
    w, g, m, v = values(n, 42)
    g = np.where(np.isfinite(g), g, F32(0.5)).astype(F32)
    master, grad = torch.from_numpy(w.copy()).cuda(), torch.from_numpy(g.copy()).cuda()
    shadow = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    word = torch.full((1,), 7, dtype=torch.int32, device="cuda")
    tr = FlatMLP(spec, master, shadow, grad, 256, optimizer="adam", lr=1.7e-3, step_dev_ptr=word.data_ptr())
    tr.m.copy_(torch.from_numpy(m))
    tr.v.copy_(torch.from_numpy(v))
    tr.optimizer_step(3)
    torch.cuda.synchronize()
    c = Case(True, n, w, g, m, v, lr=1.7e-3, step=3, word=7, zero_grad=True, label="FlatMLP adam")
    out = {"w": master.cpu().numpy(), "grad": grad.cpu().numpy(), "m": tr.m.cpu().numpy(), "v": tr.v.cpu().numpy(),
           "shadow": shadow.view(torch.int16).cpu().numpy().view(np.uint16)}
    assert_conforms(c, out, [])


# ------------------------------------------------------------------------------ binding checks
def test_optim_bindings_refuse_mismatched_buffers():
    n = 1024
    off = torch.zeros(1, dtype=torch.int32, device="cuda")
    big = {k: torch.zeros(2 * n + 16, device="cuda") for k in "wgmv"}
    sh_big = torch.zeros(n + 8, dtype=torch.bfloat16, device="cuda")
    ok = {k: t[:n] for k, t in big.items()}
    mis = {k: t[1:n + 1] for k, t in big.items()}                 # 4-byte offset
    short = {k: t[:n - 4] for k, t in big.items()}
    strided = {k: t[:2 * n:2] for k, t in big.items()}

    def plain(adam=True, step=1, **kw):
        a = {**ok, "s": sh_big[:n], **kw}
        C().optim_step(adam, a["w"], a["g"], a["s"], a["m"], a["v"], 1e-2, 0.0, 0.9, 0.999, 1e-8, step, 0,
                       off.data_ptr(), True)

    def recipe(adam=True, step=1, **kw):
        a = {**ok, "s": sh_big[:n], "ws": _ws(), **kw}
        C().optim_recipe_step(adam, a["w"], a["g"], a["s"], a["m"], a["v"], 1e-2, 0.9, 0.999, 1e-8, step, 0, 0.0,
                              None, 0, 0, 0, a["ws"], active_ptr=off.data_ptr())

    before = {k: t.clone() for k, t in big.items()}
    for fn in (plain, recipe):
        fn()
        fn(adam=False)
        bads = [dict(step=0), dict(g=short["g"]), dict(m=short["m"]), dict(v=short["v"]), dict(s=sh_big[:n - 1]),
                dict(w=mis["w"]), dict(g=mis["g"]), dict(m=mis["m"]), dict(v=mis["v"]), dict(s=sh_big[1:n + 1]),
                dict(g=strided["g"]), dict(m=strided["m"]), dict(g=ok["g"].to(torch.bfloat16)),
                dict(s=ok["w"]), dict(g=ok["g"].cpu())]
        if fn is recipe:
            wsb = torch.zeros(C().grad_norm_workspace_bytes() + 8, dtype=torch.uint8, device="cuda")
            bads += [dict(adam=False, step=0), dict(ws=wsb[4:])]
        for b in bads:
            with pytest.raises(RuntimeError):
                fn(**b)
    torch.cuda.synchronize()
    assert all(torch.equal(before[k], big[k]) for k in big)


def test_grad_norm_binding_refuses_misaligned_buffers():
    n = 1024
    off = torch.zeros(1, dtype=torch.int32, device="cuda")
    g = torch.ones(2 * n + 8, device="cuda")
    norms = torch.zeros(1, device="cuda")
    wsb = torch.zeros(C().grad_norm_workspace_bytes() + 8, dtype=torch.uint8, device="cuda")
    ws = wsb[:C().grad_norm_workspace_bytes()]
    C().grad_norm(g[:n], ws, norms, 0, 1.0, None, off.data_ptr())
    for args in ((g[1:n + 1], ws), (g[:2 * n:2], ws), (g[:n], wsb[4:])):
        with pytest.raises(RuntimeError):
            C().grad_norm(*args, norms, 0, 1.0, None, off.data_ptr())
    torch.cuda.synchronize()
    assert float(norms) == 0.0 and int(wsb.count_nonzero()) == 0


def test_cast_bindings_refuse_mismatched_buffers():
    n = 1024
    x = torch.randn(n, device="cuda")
    dst_big = torch.zeros(n + 16, dtype=torch.bfloat16, device="cuda")
    # no predicate on these two: only mismatches that stay in bounds and aligned
    for dst in (torch.zeros(n, device="cuda"), dst_big[:n + 8]):
        with pytest.raises(RuntimeError):
            C().cast_f32_to_bf16(x, dst)
    a, b = x.to(torch.bfloat16), (x * 3).to(torch.bfloat16)
    for args in ((a, b, torch.zeros(n, device="cuda")), (a, b, dst_big[:n + 8]), (a, x, dst_big[:n]),
                 (x, b, dst_big[:n])):
        with pytest.raises(RuntimeError):
            C().add_bf16(*args)
    # cast_u8_to_bf16 is predicated: undersized / misaligned buffers only with the predicate word 0
    off = torch.zeros(1, dtype=torch.int32, device="cuda")
    u = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
    C().set_predicate(off.data_ptr())
    try:
        for args in ((u[:n], dst_big[:n - 1]), (u[:n], dst_big[1:n + 1]), (u[1:n + 1], dst_big[:n]),
                     (u[:n], torch.zeros(n, device="cuda"))):
            with pytest.raises(RuntimeError):
                C().cast_u8_to_bf16(*args, 1.0)
    finally:
        C().set_predicate(0)
    torch.cuda.synchronize()
    assert int(dst_big.view(torch.int16).count_nonzero()) == 0
