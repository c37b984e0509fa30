"""DP-SGD in the persistent MLP trainer (``mlp_dpsgd_round_kernel``, driven through ``FlatMLP`` and
``FusedEngine`` with ``dpsgd_fused``) against the generic engine's definition of a DP-SGD step
(``ops/dpsgd.py``): the per-example norms of the two R = 1 sites against fp64 over the step's own bf16
rows, the clip factors against ``clip_factors`` bit for bit, the plain trainer's weights bit for bit when
nothing is clipped, the released gradient against fp64, the noise against ``dpsgd_noise``, a dropped
example, multi-step launches, the refusals and FusedEngine rounds.

The released gradient is read from the test hook ``dpsgd_dbg``: per step the rows' sq0, sq1, ab0, ab1
and c, then the last step's released gradient (noise added, before any proximal term).

A DP-SGD step has no atomics in its gradients (fixed-order norms, factors, bias sums and noise), so launches
from the same state are compared bit for bit.  ``BFLC_MLP_BMW=128`` (128-row weight-gradient tiles) is read
once per process: ``test_bm_w_128`` reruns the released-gradient and noise checks in a subprocess with it."""
import os
import subprocess
import sys
import math

import numpy as np
import pytest
import torch

from bflc_demo_b200._native import C
from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec
from bflc_demo_b200.ops.dpsgd import clip_factors, noise_sigma
from test_gpu_trainer_conformance import gamma

pytestmark = pytest.mark.gpu

D, H, NC = 784, 256, 62
WORD = 11            # the plan's optimizer-step word the noise and Adam's bias corrections read
HUGE = 1e30          # a clip above every bound: c = 1


class Setup:
    """Seeded inputs and one FlatMLP per launch from the same initial state."""

    def __init__(self, B, fp8=False, opt="sgd", rows=None, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.B, self.fp8, self.opt = B, fp8, opt
        self.rows = rows or B
        self.x_u8 = torch.randint(0, 256, (self.rows, D), generator=g, dtype=torch.uint8).cuda()
        self.x = torch.empty(self.rows, D, device="cuda", dtype=torch.bfloat16)
        self.x_dq = torch.empty_like(self.x) if fp8 else None
        C().prep_inputs(self.x_u8, self.x, None, None, 1.0 / 255.0, self.x_dq)
        self.y = torch.randint(0, NC, (self.rows,), generator=g, dtype=torch.int32).cuda()
        self.spec = mlp_spec(D, H, NC)
        self.master0 = torch.zeros(self.spec.total, device="cuda")
        self.spec.init_(self.master0, seed=seed)

    def trainer(self, clip=0.0, noise=0.0, dseed=0, prox_mu=0.0, hook_steps=None):
        master = self.master0.clone()
        self.word = torch.tensor([WORD], device="cuda", dtype=torch.int32)
        anchor = (self.master0 * 0.5) if prox_mu > 0 else None
        t = FlatMLP(self.spec, master, master.bfloat16(), torch.zeros_like(master), self.B, optimizer=self.opt,
                    lr=0.05 if self.opt == "sgd" else 1e-3, step_dev_ptr=self.word.data_ptr(), fp8=self.fp8,
                    prox_mu=prox_mu, anchor=anchor, dpsgd_clip=clip, dpsgd_noise=noise, dpsgd_seed=dseed)
        if clip > 0 and hook_steps:
            t.dpsgd_dbg = torch.zeros(hook_steps * 5 * self.B + self.spec.total, device="cuda")
        if self.fp8:
            t.quantize_weights()
        return t

    def run(self, t, steps=1, x=None, y=None, epoch_rows=0):
        bar = torch.zeros(1, device="cuda", dtype=torch.int32)
        x = self.x if x is None else x
        y = self.y if y is None else y
        t.train_epoch_fused(x, y, steps, bar.data_ptr(), x_dq=self.x_dq if self.fp8 else None, epoch_rows=epoch_rows)
        torch.cuda.synchronize()
        return t

    def hook(self, t, step=0):
        B = self.B
        r = t.dpsgd_dbg[step * 5 * B:(step + 1) * 5 * B].view(5, B).cpu().numpy()
        return r[:2], r[2:4], r[4]

    def grad_hook(self, t, steps=1):
        return t.dpsgd_dbg[steps * 5 * self.B:]


CASES = [(512, False, "sgd"), (512, False, "adam"), (512, True, "sgd"), (512, True, "adam"), (200, False, "sgd")]
IDS = [f"B{b}-{'fp8' if f else 'bf16'}-{o}" for b, f, o in CASES]


def _rows(s, t):
    B = s.B
    return (s.x[:B].double(), t.h[:B].double(), t.dlogits[:B, :NC].double(), t.dh[:B].double())


@pytest.mark.parametrize("B, fp8, opt", CASES, ids=IDS)
def test_norms_and_clip_factors(B, fp8, opt):
    """sq / ab against fp64 over the step's own bf16 rows (c = 1: the rows are stored unscaled); at a
    binding clip the same sq / ab bits and c == clip_factors(sq, ab, B, C) bit for bit."""
    s = Setup(B, fp8, opt)
    a = s.run(s.trainer(HUGE, hook_steps=1))
    sq, ab, c = s.hook(a)
    assert (c == 1).all()
    x, h, dz, dh = _rows(s, a)
    a0, b0 = (dz * dz).sum(1), (h * h).sum(1) + 1
    a1, b1 = (dh * dh).sum(1), (x * x).sum(1) + 1
    ref_sq = torch.stack([a0 * b0, a1 * b1]).cpu().numpy()
    ref_ab = torch.stack([a0.sqrt() * b0.sqrt(), a1.sqrt() * b1.sqrt()]).cpu().numpy()
    # fp32 sums of <= D + 1 terms, two products / square roots: gamma(D + 8) relative
    tol = gamma(D + 8)
    assert np.all(np.abs(sq - ref_sq) <= tol * ref_sq + 1e-30)
    assert np.all(np.abs(ab - ref_ab) <= tol * ref_ab + 1e-30)
    clip = float(np.median(np.sqrt(sq.sum(0))) * B)   # about half the examples are clipped
    b = s.run(s.trainer(clip, hook_steps=1))
    sq2, ab2, c2 = s.hook(b)
    assert np.array_equal(sq2.view(np.uint32), sq.view(np.uint32))
    assert np.array_equal(ab2.view(np.uint32), ab.view(np.uint32))
    want = clip_factors(sq, ab, B, clip)
    assert np.array_equal(c2.view(np.uint32), want.view(np.uint32))
    assert 0.2 < float((c2 < 1).mean()) < 0.8
    assert int(b.dpsgd_dropped.item()) == 0


@pytest.mark.parametrize("B, fp8, opt", CASES, ids=IDS)
def test_unclipped_step_equals_the_plain_trainer(B, fp8, opt):
    """C above every bound, z = 0: the 2-D weights equal the plain trainer's bit for bit; the biases differ
    only by the order of their column sums (fixed-order here, atomics there)."""
    s = Setup(B, fp8, opt)
    plain = s.run(s.trainer())
    dp = s.run(s.trainer(HUGE))
    for name in ("w1", "w2"):
        assert torch.equal(plain.p[name], dp.p[name]), name
    for name in ("b1", "b2"):
        d = (plain.p[name] - dp.p[name]).abs().max().item()
        scale = plain.p[name].abs().max().item() + 1.0
        assert d <= 1e-5 * scale, (name, d)


@pytest.mark.parametrize("B, fp8, opt", CASES, ids=IDS)
def test_released_gradient_against_fp64(B, fp8, opt):
    """The clipped release (z = 0) against the fp64 sum of c_n times each example's gradient over the
    step's own bf16 rows; each example's contribution is at most C / B in norm."""
    s = Setup(B, fp8, opt)
    a = s.run(s.trainer(HUGE, hook_steps=1))
    x, h, dz, dh = _rows(s, a)
    sq, _, _ = s.hook(a)
    clip = float(np.median(np.sqrt(sq.sum(0))) * B)
    b = s.run(s.trainer(clip, hook_steps=1))
    _, _, c = s.hook(b)
    cd = torch.from_numpy(c.astype(np.float64)).cuda()[:, None]
    g = s.grad_hook(b).double()
    sp = s.spec
    ref = {"w1": (dh * cd).t() @ x, "w2": (dz * cd).t() @ h, "b1": (dh * cd).sum(0), "b2": (dz * cd).sum(0)}
    mag = {"w1": (dh * cd).abs().t() @ x.abs(), "w2": (dz * cd).abs().t() @ h.abs(),
           "b1": (dh * cd).abs().sum(0), "b2": (dz * cd).abs().sum(0)}
    for name in ref:
        e = sp.by_name[name]
        out = g[e.offset:e.offset + e.numel].view(e.shape)
        # the scaled rows round to bf16 once (2^-8 relative), then fp32 sums over B rows
        bound = (2.0 ** -8 + gamma(B + 2)) * mag[name] + 1e-30
        assert bool(((out - ref[name]).abs() <= bound).all()), name
    norms = np.sqrt(sq.sum(0).astype(np.float64))
    assert np.all(c * norms <= clip / B * (1 + 1e-5))


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
def test_noise_is_dpsgd_noise_of_the_clipped_gradient(fp8):
    """z > 0: the hook's gradient is C().dpsgd_noise applied to the z = 0 gradient under the same key and word,
    bit for bit -- the generic engine's keying over the same flat layout -- and another key draws other noise."""
    s = Setup(512, fp8)
    clip, z, key = 0.5, 1.3, 0xC0FFEE1234
    g0 = s.grad_hook(s.run(s.trainer(clip, 0.0, key, hook_steps=1))).clone()
    g1 = s.grad_hook(s.run(s.trainer(clip, z, key, hook_steps=1)))
    want = g0.clone()
    C().dpsgd_noise(want, key, torch.tensor([WORD], device="cuda", dtype=torch.int32), 0,
                    float(noise_sigma(z, clip, 512)))
    # the hook covers every parameter; the padding between tensors carries no gradient
    for e in s.spec.entries:
        sl = slice(e.offset, e.offset + e.numel)
        assert torch.equal(g1[sl], want[sl]), e.name
        assert not torch.equal(g1[sl], g0[sl]), e.name
    g2 = s.grad_hook(s.run(s.trainer(clip, z, key + 1, hook_steps=1)))
    assert not torch.equal(g1, g2)


def test_dropped_example_releases_exact_zeros():
    """An example whose h overflows to inf is dropped and counted; its dz, dh and h rows are exact zeros
    and the step is finite."""
    s = Setup(512)
    s.x[3].fill_(3.0e38)
    t = s.run(s.trainer(1.0, 0.5, 7, hook_steps=1))
    _, _, c = s.hook(t)
    assert c[3] == 0 and int(t.dpsgd_dropped.item()) == 1 and np.all(c[np.arange(512) != 3] > 0)
    for buf in (t.h[3], t.dh[3], t.dlogits[3]):
        assert not bool(buf.float().abs().sum())
    assert bool(torch.isfinite(s.grad_hook(t)).all()) and bool(torch.isfinite(t.master).all())


@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_multi_step_launch_equals_single_steps(opt):
    """8 steps over an epoch of 4 batches in one launch equal 8 single-step launches (step word and rows
    advanced by hand) bit for bit, and a rerun gives the same bits."""
    B, E = 256, 4
    s = Setup(B, opt=opt, rows=E * B)
    clip, z, key = 0.3, 0.9, 99
    multi = s.run(s.trainer(clip, z, key), steps=8, epoch_rows=E * B)
    again = s.run(s.trainer(clip, z, key), steps=8, epoch_rows=E * B)
    assert torch.equal(multi.master, again.master)
    single = s.trainer(clip, z, key)
    for i in range(8):
        s.word.fill_(WORD + i)
        rows = slice((i % E) * B, (i % E + 1) * B)
        s.run(single, x=s.x[rows].contiguous(), y=s.y[rows].contiguous())
    assert torch.equal(multi.master, single.master)
    if opt == "adam":
        assert torch.equal(multi.m, single.m) and torch.equal(multi.v, single.v)


def test_refusals_before_launch():
    s = Setup(256)
    t = s.trainer(1.0)
    bar = torch.zeros(1, device="cuda", dtype=torch.int32)
    for kw in (dict(plan=0), dict(plan=3), dict(epiopt=0)):
        with pytest.raises(ValueError, match="plan 4"):
            t.train_epoch_fused(s.x, s.y, 1, bar.data_ptr(), **kw)
    with pytest.raises(ValueError, match="train_epoch_fused"):
        t.train_epoch(s.x, s.y, 1)
    with pytest.raises(ValueError, match="hidden == 256"):
        sp = mlp_spec(D, 128, NC)
        m = torch.zeros(sp.total, device="cuda")
        FlatMLP(sp, m, m.bfloat16(), torch.zeros_like(m), 256, dpsgd_clip=1.0)
    with pytest.raises(RuntimeError, match="plan 4"):   # the binding checks too
        C().mlp_round(s.x, s.y, t.master, t.shadow, t.grad, t.offsets(), t.h, t.dlogits, t.dh, t.loss_sum,
                      t.correct, bar.data_ptr(), 256, 1, D, H, NC, 0.05, False, None, None, 0, None, 3, 1,
                      dpsgd_clip=1.0, dpsgd_dropped=t.dpsgd_dropped, dpsgd_ws=t.dpsgd_ws)
    assert int(bar.item()) == 0 and int(t.dpsgd_dropped.item()) == 0


# ------------------------------------------------------------------ FusedEngine
def _engine(graph=False, dtype="bf16", optimizer="sgd", noise=1.1, seed=5, prox_mu=0.0):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    cfg = FLConfig.for_world(1, model="mlp", hidden=256, batch_size=256, samples_per_client=1024,
                             learning_rate=0.05, optimizer=optimizer, cuda_graph=graph, dtype=dtype,
                             dpsgd_clip=0.5, dpsgd_noise=noise, dpsgd_seed=seed, dpsgd_fused=True, prox_mu=prox_mu)
    return FusedEngine(cfg, femnist_like(1, 1024, seed=7, only=0)[0])


@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_engine_graph_equals_eager_and_e2e(dtype):
    eager, graph, e2e = _engine(False, dtype), _engine(True, dtype), _engine(True, dtype)
    for e in (eager, graph):
        e.capture()
        for _ in range(2):
            e.run_round()
    e2e.capture()
    for _ in range(2):
        e2e.run_round_e2e()
    torch.cuda.synchronize()
    for e in (eager, graph, e2e):
        assert e.drain_blocks() == []
        assert int(e.dpsgd.dropped.item()) == 0
    assert torch.equal(eager.global_master, graph.global_master)
    assert torch.equal(graph.global_master, e2e.global_master)


def test_engine_checkpoint_resume_and_accounting(tmp_path):
    """Checkpoint / resume with a fixed dpsgd_seed continues bit for bit (Adam moments and step word
    included), every host ledger re-executes with no mismatch, and the local epsilon is the generic engine's
    after the same rounds of the same config."""
    from bflc_demo_b200.utils.checkpoint import load_checkpoint, save_checkpoint
    a = _engine(optimizer="adam")
    a.capture()
    a.run_round()
    torch.cuda.synchronize()
    save_checkpoint(str(tmp_path / "ck"), a)
    b = _engine(optimizer="adam")
    load_checkpoint(str(tmp_path / "ck"), b)
    b.capture()
    a.run_round()
    torch.cuda.synchronize()
    assert torch.equal(a.global_master, b.global_master)
    assert a.drain_blocks() == [] and b.drain_blocks() == []
    eps, delta = a.privacy_spent_local()
    assert math.isfinite(eps) and eps > 0
    gen = _generic(optimizer="adam")
    gen.capture()            # the warm-up round, then as many rounds as a ran
    for _ in range(2):
        gen.run_round()
    torch.cuda.synchronize()
    assert gen.drain_blocks() == []
    assert (eps, delta) == gen.privacy_spent_local()


def _generic(optimizer="sgd"):
    """The generic engine's MLP under the same DP-SGD config (without the opt-in)."""
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import build_model
    cfg = FLConfig.for_world(1, model="mlp", hidden=256, batch_size=256, samples_per_client=1024,
                             learning_rate=0.05, optimizer=optimizer, dpsgd_clip=0.5, dpsgd_noise=1.1, dpsgd_seed=5)
    shard = femnist_like(1, 1024, seed=7, only=0)[0]
    return GenericFedEngine(cfg, build_model("mlp", shard.n_classes), shard)


def test_site_order_is_the_generic_mlps(monkeypatch):
    """The generic MLP's DP-SGD step records fc2 (operand h, hidden wide) before fc1 (operand x, in_dim wide):
    sq rows [fc2, fc1], the order the trainer sums sq0 + sq1 and ab0 + ab1 in."""
    from bflc_demo_b200.ops import dpsgd as Dp
    widths = []
    orig = Dp.DPSGDStep.record

    def spy(self, dz, op, gw, gb):
        widths.append((dz.shape[1], op.shape[1]))
        return orig(self, dz, op, gw, gb)

    monkeypatch.setattr(Dp.DPSGDStep, "record", spy)
    eng = _generic()
    eng.capture()
    torch.cuda.synchronize()
    assert [w[1] for w in widths[:2]] == [H, D], widths[:4]


def test_engine_update_moves_with_sigma():
    """Same data and key: the round's update at noise z differs from z = 0 by the noise, whose spread grows
    with z as sigma = z C / B predicts (SGD: lr * sigma per step, summed over the round's steps)."""
    ups = {}
    for z in (0.0, 1.0, 2.0):
        e = _engine(noise=z, seed=5)
        start = e.global_master.clone()
        e.capture()
        torch.cuda.synchronize()
        ups[z] = e.global_master.double() - start.double()
    d1, d2 = (ups[1.0] - ups[0.0]).std().item(), (ups[2.0] - ups[0.0]).std().item()
    steps = 1024 // 256
    pred = 0.05 * float(noise_sigma(1.0, 0.5, 256)) * math.sqrt(steps)
    assert 0.8 * pred < d1 < 1.25 * pred, (d1, pred)
    assert 1.8 < d2 / d1 < 2.2


@pytest.mark.skipif(os.environ.get("BFLC_MLP_BMW") == "128", reason="runs as the subprocess itself")
def test_bm_w_128():
    """The 128-row weight-gradient tiles (dp_tile's other row mapping): the released gradient against fp64 and
    the noise against dpsgd_noise, in a process started with BFLC_MLP_BMW=128."""
    env = dict(os.environ, BFLC_MLP_BMW="128")
    here = os.path.dirname(os.path.abspath(__file__))
    proc = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__),
                           "-k", "released_gradient or noise_is_dpsgd_noise"], cwd=os.path.dirname(here), env=env,
                          capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0 and " passed" in proc.stdout and "failed" not in proc.stdout, proc.stdout[-3000:]
