"""Conformance of DP-SGD in the persistent MLP trainer (``mlp_dpsgd_round_kernel``, driven through
``FlatMLP.train_epoch_fused`` with ``dpsgd_clip > 0``) at every shape the launcher accepts: batch tails
(B 32 is less than one 64-row tile, B 200 leaves an 8-row tail tile and an empty 32-row slot), 16 and 32
clusters, 57 and 64 classes (7 padding columns of the chain's 64-wide tile, none), one K-block and no
K tail, and 128-row weight-gradient tiles (in_dim 2048 on a 132-SM part), in bf16 and fp8, under SGD
and Adam, with and without FedProx.

Each case checks, from the step's own stored rows:

a. with C above every bound and z = 0, the weights and the stored h / dlogits / dh of the plain trainer
   bit for bit, and the biases within the bound for a change of summation order;
b. the per-row norms of the test hook against fp64 (x is nonzero in its K tail, the largest |dz| of
   half the rows sits in class C - 1);
c. the clip factors against ``clip_factors`` bit for bit, at a clip that scales 20-80 % of the rows;
d. the stored rows: exactly bf16(row * c) of the unclipped rows, a dropped example's rows zero;
e. the certified bound ``B ||c_n g_n|| <= C`` in fp64 from the rows the weight gradients were built
   from (bf16 x and h, the stored dz' and dh'), with no tolerance;
f. the release: weights within gamma(B) of the fp64 sum, the biases in the kernel's fixed slot order
   bit for bit, the noise ``dpsgd_noise`` of the z = 0 release bit for bit, nothing in the padding;
g. the applied update: SGD exactly (fp32 spec, FedProx term included), Adam within the trainer suite's
   bound, the shadow bf16(master'), the gradient buffer zero, fp8 weights re-quantised from master';
h. FedProx leaves the release bit for bit unchanged (the noise comes first).

Then multi-step launches against single-step replay, dropped examples at tile and cluster edges, and
the refusals: class counts outside 57..64 (DP-SGD and fp8) and batches beyond what plan 4 can hold are
refused by FlatMLP and FusedEngine before anything launches, and ``mlp_round_plan`` answers as the
launcher decides.

The checking functions are numpy helpers that need no GPU; ``test_dpsgd_fused_host.py`` requires each
modelled shape mistake to fail its helper.
"""
import numpy as np
import pytest
import torch

from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec
from bflc_demo_b200.ops.dpsgd import clip_factors, noise_sigma
from test_gpu_trainer_conformance import (LR, Run, adam_slack, allowed_plans, check_one_step, expected_bm_w,
                                          gamma, int_fixture, ran_plan, real_fixture, sms)
from test_gpu_layer_conformance import assert_bound

F32, F64 = np.float32, np.float64
HUGE = 1e30          # a clip above every bound: c = 1
KEY = 0xD95E7C41A3   # the noise key of every noised run
Z = 1.1              # the noise multiplier of every noised run
MU = 0.25            # FedProx
BASE = 7             # Adam's carried step word


# ------------------------------------------------------------------ numpy helpers (no GPU)
def _bf16(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=F32)).to(torch.bfloat16).float().numpy()


def _sq(a):
    return (np.asarray(a, F64) ** 2).sum(1)


def check_norms(sq, ab, x, h, dz, dh):
    """The hook's sq0, sq1, ab0, ab1 (fp32 [2, B] each) against fp64 over the step's bf16 rows: x [B, D],
    h [B, 256], dz [B, C] (the real classes), dh [B, 256]; fp32 sums of at most D + 1 terms and two
    products / square roots, gamma(D + 8) relative.  The build flushes subnormals (-ftz): each of a row's
    n squares and partial sums may lose up to 2^-126, so a = ||dz||^2 (||dh||^2) is also within n 2^-126
    absolute, sq within that times b and sqrt(a) within its square root (a saturated row's dz underflows)."""
    a0, b0 = _sq(dz), _sq(h) + 1
    a1, b1 = _sq(dh), _sq(x) + 1
    ref_sq = np.stack([a0 * b0, a1 * b1])
    ref_ab = np.stack([np.sqrt(a0) * np.sqrt(b0), np.sqrt(a1) * np.sqrt(b1)])
    tol = gamma(x.shape[1] + 8)
    ea = np.array([[2 * dz.shape[1] * 2.0 ** -126], [2 * dh.shape[1] * 2.0 ** -126]])
    b = np.stack([b0, b1])
    ftz = {"sq": ea * b * (1 + tol), "ab": np.sqrt(ea) * np.sqrt(b) * (1 + tol)}
    for name, got, ref in (("sq", sq, ref_sq), ("ab", ab, ref_ab)):
        bad = ~(np.abs(np.asarray(got, F64) - ref) <= tol * ref + ftz[name])
        assert not bad.any(), f"{name}: {int(bad.sum())} rows off fp64, first {np.argwhere(bad)[:4].tolist()}"


def check_clip_factors(c, sq, ab, clip):
    want = clip_factors(sq, ab, sq.shape[1], clip)
    assert np.array_equal(np.asarray(c, F32).view(np.uint32), want.view(np.uint32)), "c != clip_factors(sq, ab)"


def check_stored_rows(c, rows0, rows1):
    """rows0 = (h, dz, dh) of the unclipped step (c = 1), rows1 the clipped step's stored rows: dz' and
    dh' are bf16(row * c) exactly, +0 where c = 0; h is unchanged, and zero where c = 0."""
    c = np.asarray(c, F32)
    zero = c == 0
    h0, dz0, dh0 = rows0
    h1, dz1, dh1 = rows1
    for name, r0, r1 in (("dz", dz0, dz1), ("dh", dh0, dh1)):
        with np.errstate(all="ignore"):
            want = _bf16(np.asarray(r0, F32) * c[:, None])
        want[zero] = 0
        assert np.array_equal(np.asarray(r1, F32).view(np.uint32), want.view(np.uint32)), \
            f"stored {name} != bf16({name} * c): rows {np.unique(np.argwhere(r1 != want)[:, 0])[:8].tolist()}"
    want_h = np.asarray(h0, F32).copy()
    want_h[zero] = 0
    assert np.array_equal(np.asarray(h1, F32).view(np.uint32), want_h.view(np.uint32)), "stored h"


def certified_norms(x, h, dz, dh):
    """fp64 norm of each example's contribution to the release, from the rows the GEMMs multiply."""
    with np.errstate(all="ignore"):
        return np.sqrt(_sq(dz) * (_sq(h) + 1) + _sq(dh) * (_sq(x) + 1))


def check_certified_bound(x, h, dz, dh, clip):
    """B ||R_n|| <= C for every example, exactly (DESIGN's certified clip)."""
    B = x.shape[0]
    n = certified_norms(x, h, dz, dh)
    ok = n * B <= float(F32(clip))
    assert ok.all(), (f"{int((~ok).sum())} examples above C / B: worst B ||R|| / C = "
                      f"{np.nanmax(n * B / float(F32(clip)))}, rows {np.argwhere(~ok)[:8, 0].tolist()}")


def check_padding(v, spec, what):
    pad = np.ones(spec.total, bool)
    for e in spec.entries:
        pad[e.offset:e.offset + e.numel] = False
    assert not np.asarray(v)[pad].any(), f"{what}: nonzero padding between tensors"


def check_release(g, x, h, dz, dh, spec):
    """The z = 0 release against the step's stored rows: dW1 = dh'^T x and dW2 = dz'^T h within gamma(B + 2)
    of fp64; db1 / db2 the fixed-order slot sums of the stored rows bit for bit; zero padding."""
    from test_dpsgd_fused_host import fixed_colsum
    B = x.shape[0]
    g = np.asarray(g, F32)
    x64, h64, dz64, dh64 = (np.asarray(a, F64) for a in (x, h, dz, dh))
    ref = {"w1": (dh64.T @ x64, np.abs(dh64).T @ np.abs(x64)), "w2": (dz64.T @ h64, np.abs(dz64).T @ np.abs(h64))}
    for name, (r, mag) in ref.items():
        e = spec.by_name[name]
        out = g[e.offset:e.offset + e.numel].reshape(e.shape).astype(F64)
        bad = ~(np.abs(out - r) <= gamma(B + 2) * mag + 1e-30)
        assert not bad.any(), f"released {name}: {int(bad.sum())} elements off fp64"
    n_tiles = -(-B // 64)
    for name, rows in (("b1", dh), ("b2", dz)):
        e = spec.by_name[name]
        want = fixed_colsum(np.asarray(rows, F32), n_tiles)
        got = g[e.offset:e.offset + e.numel]
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"released {name} != fixed-order slot sums"
    check_padding(g, spec, "release")


def sgd_spec(w, g, lr, anchor=None, mu=0.0):
    """master' of the optimizer epilogue: g' = fma(mu, w - anchor, g) under FedProx, then w - lr g'
    (either rounding: the product rounded first, or one fma), subnormals flushed to zero as the build's
    -ftz does."""
    from test_optim_spec_host import f32_fma, f32_mul, f32_sub, ftz
    w, g = np.asarray(w, F32), np.asarray(g, F32)
    if mu > 0:
        g = f32_fma(F32(mu), f32_sub(w, np.asarray(anchor, F32)), g)
    lr = F32(lr)
    unfused = f32_sub(w, f32_mul(lr, g))
    fused = f32_fma(-lr, g, w)
    return unfused, fused, g


# ------------------------------------------------------------------ the case matrix
def _cases():
    out = []
    for dt in ("bf16", "fp8"):
        for o in ("sgd", "adam"):
            out.append((512, 784, 62, dt, o))
    shapes = [(32, 784, 62), (128, 784, 62), (200, 784, 62), (1024, 784, 62), (2048, 784, 62),
              (256, 784, 57), (256, 784, 64), (256, 64, 62), (256, 512, 62), (256, 2048, 62)]
    for B, D, C in shapes:
        for dt in ("bf16", "fp8"):
            if dt == "fp8" and (B % 128 or D % 16):
                continue
            for o in ("sgd", "adam"):
                out.append((B, D, C, dt, o))
    return out


CASES = _cases()
IDS = [f"B{b}-{d}x256x{c}-{dt}-{o}" for b, d, c, dt, o in CASES]
# grids beyond the 16 resident clusters the trainer suite assumes: refused cleanly or run and conform
MAY_REFUSE = {(2048, 784), (256, 2048)}


def fixture(B, D, C, opt, seed=0):
    """SGD on the integer fixture, Adam on the real one; half the rows labelled C - 1 (so that the largest
    |dz| of those rows sits in the last class) and every row nonzero somewhere in the K tail."""
    fx = (int_fixture if opt == "sgd" else real_fixture)(D, 256, C, B, seed=seed + B + D + C)
    y = fx.y.clone()
    y[1::2] = C - 1
    xu8 = fx.xu8.clone()
    xu8[:, D - 1] = np.uint8(255)
    return fx._replace(y=y, xu8=xu8)


class DpRun(Run):
    """Run's inputs and initial state, with a DP-SGD trainer (and the dpsgd_dbg hook) in place of the plain
    one; Adam starts from Run's warm moments and step word BASE."""

    def __init__(self, fx, fp8, opt, clip, z=0.0, mu=0.0, steps=1):
        base = BASE if opt == "adam" else 0
        super().__init__(fx, fp8, opt, base=base, moments_seed=(17 if opt == "adam" else None))
        old = self.tr
        master = fx.master.cuda().clone()
        self.anchor = (master * 0.5).contiguous() if mu > 0 else None
        self.tr = FlatMLP(self.spec, master, master.bfloat16(), torch.zeros_like(master), self.B, optimizer=opt,
                          lr=LR[opt], fp8=fp8, step_dev_ptr=self.step.data_ptr(), prox_mu=mu, anchor=self.anchor,
                          dpsgd_clip=clip, dpsgd_noise=z, dpsgd_seed=KEY)
        if opt == "adam":
            self.tr.m.copy_(old.m)
            self.tr.v.copy_(old.v)
        if fp8:
            self.tr.quantize_weights()
        self.tr.dpsgd_dbg = torch.zeros(steps * 5 * self.B + self.spec.total, device="cuda")
        self.before = {"master": master.clone(), "m": None if opt == "sgd" else self.tr.m.clone(),
                       "v": None if opt == "sgd" else self.tr.v.clone()}

    def hook(self, step=0):
        B = self.B
        r = self.tr.dpsgd_dbg[step * 5 * B:(step + 1) * 5 * B].view(5, B).cpu().numpy()
        return r[:2], r[2:4], r[4]

    def grad_hook(self, steps=1):
        return self.tr.dpsgd_dbg[steps * 5 * self.B:].clone()

    def rows(self):
        """x (bf16, what dW1 reads), h, dz (real classes), dh of the last step as numpy fp32."""
        tr, B, C = self.tr, self.B, self.fx.C
        return tuple(t.float().cpu().numpy() for t in (self.xb[:B], tr.h[:B], tr.dlogits[:B, :C], tr.dh[:B]))


def _query(B, D, C, fp8, prox):
    from bflc_demo_b200._native import C as native
    return native().mlp_round_plan(B, D, 256, C, fp8=fp8, dpsgd=True, prox=prox)


def _check_update(run, g, info):
    """(g): master' from the hook's release, the shadow, the zeroed gradient buffer, fp8's work copies."""
    tr, spec, opt = run.tr, run.spec, run.opt
    w0 = run.before["master"].cpu().numpy()
    w1 = tr.master.cpu().numpy()
    anchor = run.anchor.cpu().numpy() if run.anchor is not None else None
    mu = tr.prox_mu
    gn = g.cpu().numpy()
    if opt == "sgd":
        unfused, fused, _ = sgd_spec(w0, gn, LR["sgd"], anchor, mu)
        ok = (w1.view(np.uint32) == unfused.view(np.uint32)) | (w1.view(np.uint32) == fused.view(np.uint32))
        for e in spec.entries:
            sl = slice(e.offset, e.offset + e.numel)
            assert ok[sl].all(), f"SGD {e.name}: {int((~ok[sl]).sum())} elements off the fp32 spec ({info})"
    else:
        from test_optim_spec_host import f32_fma, f32_sub
        gp = gn if mu == 0 else f32_fma(F32(mu), f32_sub(w0, anchor), gn)
        gt = torch.from_numpy(np.asarray(gp, F64))
        m0, v0 = run.before["m"].double().cpu(), run.before["v"].double().cpu()
        (w, m, v), (sw, sm, sv) = adam_slack(torch.from_numpy(w0.astype(F64)), m0, v0, gt, torch.zeros_like(gt),
                                             F64(F32(LR["adam"])), BASE + 1)
        for e in spec.entries:
            sl = slice(e.offset, e.offset + e.numel)
            assert_bound(tr.m.cpu()[sl], m[sl], sm[sl], f"Adam m {e.name} ({info})")
            assert_bound(tr.v.cpu()[sl], v[sl], sv[sl], f"Adam v {e.name} ({info})")
            assert_bound(tr.master.cpu()[sl], w[sl], sw[sl], f"Adam w {e.name} ({info})")
    check_padding(w1, spec, f"master' ({info})")
    assert torch.equal(tr.shadow, tr.master.bfloat16()), f"shadow != bf16(master') ({info})"
    assert int(torch.count_nonzero(tr.grad)) == 0, f"gradient buffer not re-zeroed ({info})"
    if run.fp8:
        q, dq = tr.work_q.clone(), tr.work_dq.clone()
        tr.quantize_weights()
        torch.cuda.synchronize()
        L, D, H = tr.ql, tr.in_dim, tr.hidden
        for name, nbytes in (("w1q", H * D), ("w1sf", -(-H // 128) * L["kb1"] * 512), ("w2q", 64 * H),
                             ("w2sf", L["kb2"] * 512)):
            sl = slice(L[name], L[name] + nbytes)
            assert torch.equal(q[sl], tr.work_q[sl]), f"work_q {name} not re-quantised from master' ({info})"
        assert torch.equal(dq, tr.work_dq), f"work_dq not re-quantised from master' ({info})"


# ------------------------------------------------------------------ GPU: one step at every shape
@pytest.mark.gpu
@pytest.mark.parametrize("B,D,C,dtype,opt", CASES, ids=IDS)
def test_one_step_conforms(B, D, C, dtype, opt):
    fp8 = dtype == "fp8"
    fx = fixture(B, D, C, opt)
    q = _query(B, D, C, fp8, False)
    qp = _query(B, D, C, fp8, True)
    assert q["ok"] == qp["ok"], (q, qp)
    if not q["ok"]:
        assert (B, D) in MAY_REFUSE, q
        for mu in (0.0, MU):
            with pytest.raises(ValueError, match="phase plan 4"):
                DpRun(fx, fp8, opt, 1.0, mu=mu)
        print(f"[dpsgd conformance] B={B} {D}-256-{C} {dtype} {opt}: refused at construction "
              f"({q['error'] or qp['error']}, {q['max_clusters']} resident clusters on {sms()} SMs)")
        return
    assert q["plan"] == 4 and q["bm_w"] == expected_bm_w(D, 256), q

    # (a) unclipped, z = 0, against the plain trainer
    plain = Run(fx, fp8, opt, base=BASE if opt == "adam" else None, moments_seed=(17 if opt == "adam" else None))
    plain.launch(4, 1, 1)
    u = DpRun(fx, fp8, opt, HUGE)
    u.launch(-1, -1, 1)
    got_plan, _ = ran_plan(u.dbg.cpu()[0])
    assert got_plan == 4 and got_plan in allowed_plans(4, D, 256, C, B), got_plan
    info = f"plan {got_plan}, bm_w {q['bm_w']}, grid {q['grid']} on {sms()} SMs"
    for name in ("w1", "w2"):
        assert torch.equal(plain.tr.p[name], u.tr.p[name]), f"unclipped {name} != plain ({info})"
    for name in ("h", "dlogits", "dh"):
        assert torch.equal(getattr(plain.tr, name), getattr(u.tr, name)), f"unclipped {name} != plain ({info})"
    sq, ab, c1 = u.hook()
    assert (c1 == 1).all()
    x, h0, dz0, dh0 = u.rows()
    g_u = u.grad_hook()
    check_release(g_u.cpu().numpy(), x, h0, dz0, dh0, u.spec)
    _check_update(u, g_u, info)
    # the biases (SGD: linear in the gradient): the plain trainer sums the fp32 rows by atomics, the DP path
    # their bf16 copies in a fixed order -- two summation orders plus the rows' bf16 rounding apart
    if opt == "sgd":
        for name, rows in (("b1", dh0), ("b2", dz0)):
            mag = np.abs(rows.astype(F64)).sum(0)
            wd = u.tr.p[name].double().cpu().numpy()
            d = np.abs(plain.tr.p[name].double().cpu().numpy() - wd)
            slack = F64(F32(LR["sgd"])) * (2.0 ** -8 + 2 * gamma(B)) * mag * (1 + 1e-6) + 2.0 ** -22 * np.abs(wd)
            assert (d <= slack).all(), f"bias {name} plain vs DP: {d.max()} ({info})"

    # (b) norms, (c) clip factors at a binding clip
    check_norms(sq, ab, x, h0, dz0, dh0)
    clip = float(np.median(np.sqrt(sq.astype(F64).sum(0))) * B)
    k = DpRun(fx, fp8, opt, clip)
    k.launch(-1, -1, 1)
    sq2, ab2, c = k.hook()
    assert np.array_equal(sq2.view(np.uint32), sq.view(np.uint32)) and np.array_equal(ab2.view(np.uint32), ab.view(np.uint32))
    check_clip_factors(c, sq, ab, clip)
    frac = float((c < 1).mean())
    assert 0.2 < frac < 0.8, frac
    assert int(k.tr.dpsgd_dropped.item()) == 0
    # (d) stored rows, (e) the certified bound, (f) the release, (g) the update
    _, h1, dz1, dh1 = k.rows()
    check_stored_rows(c, (h0, dz0, dh0), (h1, dz1, dh1))
    check_certified_bound(x, h1, dz1, dh1, clip)
    g0 = k.grad_hook()
    check_release(g0.cpu().numpy(), x, h1, dz1, dh1, k.spec)
    _check_update(k, g0, info)

    # (f) noise: dpsgd_noise of the z = 0 release; (g) its update; (h) FedProx leaves the release alone
    from bflc_demo_b200._native import C as native
    n = DpRun(fx, fp8, opt, clip, z=Z)
    n.launch(-1, -1, 1)
    gz = n.grad_hook()
    want = g0.clone()
    word = BASE if opt == "adam" else 0
    native().dpsgd_noise(want, KEY, torch.tensor([word], device="cuda", dtype=torch.int32), 0,
                         float(noise_sigma(Z, clip, B)))
    for e in n.spec.entries:
        sl = slice(e.offset, e.offset + e.numel)
        assert torch.equal(gz[sl], want[sl]), f"noise on {e.name} != dpsgd_noise ({info})"
    check_padding(gz.cpu().numpy(), n.spec, f"noised release ({info})")
    _check_update(n, gz, info)
    p = DpRun(fx, fp8, opt, clip, z=Z, mu=MU)
    p.launch(-1, -1, 1)
    assert ran_plan(p.dbg.cpu()[0])[0] == 4
    assert torch.equal(p.tr.dpsgd_dbg, n.tr.dpsgd_dbg), f"FedProx changed the release ({info})"
    _check_update(p, p.grad_hook(), info + ", FedProx")
    print(f"[dpsgd conformance] B={B} {D}-256-{C} {dtype} {opt}: {info}, {frac:.0%} clipped, conforms")


# the plain trainer at the shapes its own suite does not run, so that (a) rests on a checked step
@pytest.mark.gpu
@pytest.mark.parametrize("B,D,C,opt", [(32, 784, 62, "sgd"), (32, 784, 62, "adam"), (256, 784, 57, "sgd"),
                                       (256, 784, 57, "adam"), (256, 2048, 62, "sgd"), (256, 2048, 62, "adam")])
def test_plain_trainer_at_the_dp_only_shapes(B, D, C, opt):
    fx = (int_fixture if opt == "sgd" else real_fixture)(D, 256, C, B, seed=B + D + C)
    check_one_step(fx, False, 4, 1, opt, BASE if opt == "adam" else None)


# ------------------------------------------------------------------ multi-step launches
MULTI = [(32, "bf16", "sgd"), (200, "bf16", "sgd"), (1024, "bf16", "sgd"), (512, "fp8", "adam")]


@pytest.mark.gpu
@pytest.mark.parametrize("mu", [0.0, MU], ids=["noprox", "prox"])
@pytest.mark.parametrize("B,dtype,opt", MULTI, ids=[f"B{b}-{d}-{o}" for b, d, o in MULTI])
def test_steps_in_one_launch_equal_single_step_replay(B, dtype, opt, mu):
    """S = 3 steps over E = 2 batches in one launch against three single-step launches (rows and step word
    advanced by hand), bit for bit: master, shadow, moments, the last step's hook."""
    fp8, S, E = dtype == "fp8", 3, 2
    D, C = 784, 62
    fx = fixture(E * B, D, C, opt)._replace(B=B)
    clip = 0.05
    multi = DpRun(fx, fp8, opt, clip, z=Z, mu=mu, steps=S)
    multi.bar.zero_()
    multi.tr.train_epoch_fused(multi.xb, multi.y, S, multi.bar.data_ptr(), plan=-1,
                               **({"x_dq": multi.x_dq} if fp8 else {}), epoch_rows=E * B)
    torch.cuda.synchronize()
    one = DpRun(fx, fp8, opt, clip, z=Z, mu=mu)
    base = BASE if opt == "adam" else 0
    for s in range(S):
        one.step.fill_(base + s)
        one.launch(-1, -1, 1, row0=(s % E) * B)
        _, _, c = one.hook()
        _, _, cm = multi.hook(s)
        assert np.array_equal(c.view(np.uint32), cm.view(np.uint32)), f"step {s} clip factors"
    for name in ("master", "shadow") + (("m", "v") if opt == "adam" else ()):
        assert torch.equal(getattr(multi.tr, name), getattr(one.tr, name)), name
    assert torch.equal(multi.grad_hook(S), one.grad_hook(1)), "last step's release"
    assert 0 < float((c < 1).mean()) and int(multi.tr.dpsgd_dropped.item()) == 0
    print(f"[dpsgd replay] B={B} {dtype} {opt} mu={mu}: bit-equal")


# ------------------------------------------------------------------ dropped examples at the edges
@pytest.mark.gpu
def test_dropped_examples_at_tile_and_cluster_edges():
    """Rows 0, 63, 64 (the next cluster's first) and 199 (the tail tile's last) of B 200 overflow on step 2
    of 3: their c is 0 and their rows zero, dpsgd_dropped counts them, the step is finite, and every other
    example's c is that of the run without the bad rows."""
    B, S, D, C = 200, 3, 784, 62
    bad = [0, 63, 64, 199]
    fx = fixture(S * B, D, C, "sgd")._replace(B=B)
    runs = []
    for poison in (False, True):
        r = DpRun(fx, False, "sgd", 0.05, z=Z, steps=S)
        if poison:
            r.xb[2 * B + torch.tensor(bad, device="cuda")] = 3.0e38
        r.bar.zero_()
        r.tr.train_epoch_fused(r.xb, r.y, S, r.bar.data_ptr(), plan=-1)
        torch.cuda.synchronize()
        runs.append(r)
    clean, hit = runs
    for s in range(S):
        _, _, c0 = clean.hook(s)
        _, _, c1 = hit.hook(s)
        keep = np.ones(B, bool)
        if s == 2:
            keep[bad] = False
            assert (c1[bad] == 0).all(), c1[bad]
        assert np.array_equal(c0[keep].view(np.uint32), c1[keep].view(np.uint32)), f"step {s}"
    assert int(hit.tr.dpsgd_dropped.item()) == len(bad)
    for name in ("h", "dh", "dlogits"):
        assert not bool(getattr(hit.tr, name)[bad].float().abs().sum()), name
    assert bool(torch.isfinite(hit.grad_hook(S)).all()) and bool(torch.isfinite(hit.tr.master).all())


# ------------------------------------------------------------------ refusals before launch
def _engine(n_classes, dtype="bf16", dpsgd=True, batch=256, rows=1024):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    kw = dict(dpsgd_clip=0.5, dpsgd_noise=1.0, dpsgd_fused=True) if dpsgd else {}
    cfg = FLConfig.for_world(1, model="mlp", hidden=256, batch_size=batch, samples_per_client=rows,
                             learning_rate=0.05, dtype=dtype, **kw)
    return FusedEngine(cfg, femnist_like(1, rows, seed=7, n_classes=n_classes, only=0)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("C", [2, 10, 56])
@pytest.mark.parametrize("mode", ["dpsgd", "fp8"])
def test_class_counts_outside_the_chain_refused(C, mode):
    from bflc_demo_b200 import _native
    spec = mlp_spec(784, 256, C)
    m = torch.zeros(spec.total, device="cuda")
    kw = dict(dpsgd_clip=1.0) if mode == "dpsgd" else dict(fp8=True)
    n0 = _native.C().launch_count()
    with pytest.raises(ValueError, match="57..64 classes"):
        FlatMLP(spec, m, m.bfloat16(), torch.zeros_like(m), 256, **kw)
    with pytest.raises(ValueError, match="57..64 classes"):
        _engine(C, dtype="fp8" if mode == "fp8" else "bf16", dpsgd=mode == "dpsgd")
    assert _native.C().launch_count() == n0
    # the launcher refuses them too (a host-side refusal: nothing is launched)
    assert not _query(256, 784, C, mode == "fp8", False)["ok"]


@pytest.mark.gpu
@pytest.mark.parametrize("B", [2176, 4096])
def test_batches_beyond_the_plan4_grid_refused(B):
    """Plan-4 grids of ceil(B / 64) clusters of four beyond the SM count: FlatMLP and FusedEngine refuse
    them; the launcher, called past FlatMLP's check, refuses them before launching."""
    assert -(-B // 64) * 4 > sms()
    assert not _query(B, 784, 62, False, False)["ok"]
    spec = mlp_spec(784, 256, 62)
    m = torch.zeros(spec.total, device="cuda")
    with pytest.raises(ValueError, match="phase plan 4"):
        FlatMLP(spec, m, m.bfloat16(), torch.zeros_like(m), B, dpsgd_clip=1.0)
    with pytest.raises(ValueError, match="phase plan 4"):
        _engine(62, batch=B, rows=B)
    fx = real_fixture(784, 256, 62, B, seed=3)
    run = Run(fx, False, "sgd")
    t = run.tr
    t.dpsgd_clip, t.dpsgd_sigma, t.dpsgd_seed = 1.0, 0.0, 0
    t.dpsgd_dropped = torch.zeros(1, device="cuda", dtype=torch.int32)
    t.dpsgd_ws = torch.zeros(2 * (-(-B // 64)), 256 + 64, device="cuda")
    before = t.master.clone()
    with pytest.raises(RuntimeError, match="mlp_round_sm100"):
        run.launch(-1, -1, 1)
    torch.cuda.synchronize()
    assert int(run.bar.item()) == 0 and torch.equal(t.master, before)


@pytest.mark.gpu
@pytest.mark.parametrize("B,D,C,dtype,opt", [c for c in CASES if c[4] == "sgd"],
                         ids=[i for c, i in zip(CASES, IDS) if c[4] == "sgd"])
def test_query_is_the_launchers_decision(B, D, C, dtype, opt):
    """Where the query accepts, the launch runs plan 4 with its tile height (the stamps); where it refuses,
    the launcher, called past FlatMLP's check, refuses too."""
    fp8 = dtype == "fp8"
    q = _query(B, D, C, fp8, False)
    fx = fixture(B, D, C, opt)
    if q["ok"]:
        r = DpRun(fx, fp8, opt, 1.0)
        r.launch(-1, -1, 1)
        assert ran_plan(r.dbg.cpu()[0])[0] == q["plan"] == 4
        assert q["bm_w"] == expected_bm_w(D, 256)
        return
    run = Run(fx, fp8, opt)
    t = run.tr
    t.dpsgd_clip, t.dpsgd_sigma, t.dpsgd_seed = 1.0, 0.0, 0
    t.dpsgd_dropped = torch.zeros(1, device="cuda", dtype=torch.int32)
    t.dpsgd_ws = torch.zeros(2 * (-(-B // 64)), 256 + 64, device="cuda")
    with pytest.raises(RuntimeError, match="mlp_round_sm100"):
        run.launch(-1, -1, 1)
    torch.cuda.synchronize()
    assert int(run.bar.item()) == 0
