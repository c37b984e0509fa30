"""FedProx local training on the GPU: the flat optimizer's recipe kernel against the exact fp32 model of
``test_prox_host.py``, the persistent trainer (every phase plan, optimizer placement, dtype and
optimizer) and the engines, whose anchor must be the global model the round started from."""
import numpy as np
import pytest
import torch

from test_gpu_optim_conformance import C, _ws, bf16_buf, bf16_out, f32_buf, f32_out
from test_gpu_trainer_conformance import LR, Run, allowed_plans, expected_bm_w, ran_plan, sat_fixture
from test_optim_spec_host import F32, SH_INIT, adam_w_bound, check_update, first_bad, same_bits
from test_prox_host import MU, prox_cases, prox_update

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------ flat optimizer
def launch_prox(c, anchor, mu, active=None):
    """Case c through optim_recipe_step with an anchor, on NaN-canaried buffers."""
    n, bad = c.n, []
    W, G, A = f32_buf(c.w), f32_buf(c.g), f32_buf(anchor)
    M, V = (f32_buf(c.m), f32_buf(c.v)) if c.adam else (None, None)
    SH = bf16_buf(n)
    word = torch.tensor([c.word], dtype=torch.int32, device="cuda") if c.word is not None else None
    mask = torch.from_numpy(c.mask).cuda() if c.mask is not None else None
    ws = _ws(c.coef, c.nonfinite) if c.clip == "header" else None
    mv = (M[:n], V[:n]) if c.adam else (None, None)
    C().optim_recipe_step(c.adam, W[:n], G[:n], SH[:n], *mv, c.lr, c.b1, c.b2, c.eps, c.step,
                          word.data_ptr() if word is not None else 0, c.decay, mask, c.schedule, c.W, c.T, ws,
                          active_ptr=active.data_ptr() if active is not None else 0, zero_grad=c.zero_grad,
                          anchor=A[:n], prox_mu=mu)
    torch.cuda.synchronize()
    out = {"w": f32_out(W, n, "w", bad), "grad": f32_out(G, n, "grad", bad), "shadow": bf16_out(SH, n, "shadow", bad)}
    out["m"], out["v"] = (f32_out(M, n, "m", bad), f32_out(V, n, "v", bad)) if c.adam else (c.m, c.v)
    a_after = f32_out(A, n, "anchor", bad)
    if not same_bits(a_after, anchor).all():
        bad.append("anchor written")
    return out, [f"{c.label} {b}" for b in bad]


@pytest.mark.parametrize("n", [1, 3, 4099, 100004])
@pytest.mark.parametrize("adam", [False, True], ids=["sgd", "adam"])
def test_recipe_step_with_anchor(adam, n):
    """SGD bit for bit, Adam moments bit for bit and weights within adam_w_bound, against the model;
    with and without a clip coefficient, with decay, and the skipped step (weights, moments and
    anchor untouched)."""
    for c, a in prox_cases(adam, n):
        out, bad = launch_prox(c, a, MU)
        bad += check_update(c, out, spec=prox_update(c, a, MU))
        assert not bad, "\n".join(bad[:12])


@pytest.mark.parametrize("adam", [False, True], ids=["sgd", "adam"])
def test_recipe_step_with_anchor_predicate_off_changes_nothing(adam):
    c, a = prox_cases(adam, 4099)[0]
    out, bad = launch_prox(c, a, MU, active=torch.zeros(1, dtype=torch.int32, device="cuda"))
    for k in ("w", "grad", "m", "v"):
        ok = same_bits(out[k], getattr(c, {"grad": "g"}.get(k, k)))
        bad += [] if ok.all() else [f"{k} changed at {first_bad(ok)}"]
    bad += [] if (out["shadow"] == SH_INIT).all() else ["shadow written"]
    assert not bad, bad


def test_recipe_step_refuses_a_bad_anchor():
    """Shape, dtype, alignment and mu are checked before launch; the predicate word is 0, so a missing
    check could not touch memory either."""
    n = 4099
    w = torch.zeros(n + 8, device="cuda")
    g = torch.zeros(n, device="cuda")
    off = torch.zeros(1, dtype=torch.int32, device="cuda")
    kw = dict(active_ptr=off.data_ptr())
    args = (False, w[:n], g, None, None, None, 0.1, 0.9, 0.999, 1e-8, 1, 0, 0.0, None, 0, 0, 0, None)
    bad = [dict(anchor=torch.zeros(n - 1, device="cuda"), prox_mu=0.5),
           dict(anchor=torch.zeros(n, device="cuda", dtype=torch.float64), prox_mu=0.5),
           dict(anchor=torch.zeros(n + 1, device="cuda")[1:], prox_mu=0.5),
           dict(anchor=None, prox_mu=0.5),
           dict(anchor=torch.zeros(n, device="cuda"), prox_mu=-0.5),
           dict(anchor=torch.zeros(n, device="cuda"), prox_mu=float("nan"))]
    for b in bad:
        with pytest.raises(RuntimeError):
            C().optim_recipe_step(*args, **kw, **b)
    C().optim_recipe_step(*args, **kw, anchor=torch.zeros(n, device="cuda"), prox_mu=0.5)
    C().optim_recipe_step(*args, **kw, anchor=None, prox_mu=0.0)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------ persistent trainer
TRAINER = [(d, p, eo, o) for d in ("bf16", "fp8") for p in (0, 3, 4) for eo in (0, 1) for o in ("sgd", "adam")
           if d == "bf16" or (p != 0 and eo == 1)]
TRAINER_SHAPES = [(512, 784, 256, 62), (32, 784, 256, 62)]   # the bench shape and a batch tail
# hidden 640: dW1's 64-row tiles would need more CTAs than an H100 has SMs, so the launcher takes 128-row
# weight-gradient tiles, whose FedProx pass stages only the anchor and reads the master from L2
WIDE = [("bf16", 0, eo, o, 512, 784, 640, 62) for eo in (0, 1) for o in ("sgd", "adam")]


def _run(fx, fp8, opt, mu, anchor):
    r = Run(fx, fp8, opt)
    r.tr.prox_mu, r.tr.anchor = (mu, anchor) if mu > 0 else (0.0, None)
    return r


def _step(fx, fp8, opt, plan, epiopt, mu, anchor):
    r = _run(fx, fp8, opt, mu, anchor)
    r.launch(plan, epiopt, 1)
    plans = ran_plan(r.dbg.cpu()[0])
    assert plans[0] in allowed_plans(plan, fx.D, fx.H, fx.C, fx.B) and plans[1] == epiopt, plans
    return r.state()


def _cases():
    out = []
    for d, p, eo, o in TRAINER:
        for B, D, H, Cn in TRAINER_SHAPES:
            if d == "fp8" and B % 128:
                continue
            out.append((d, p, eo, o, B, D, H, Cn))
    return out + WIDE


@pytest.mark.parametrize("dtype,plan,epiopt,opt,B,D,H,Cn", _cases(),
                         ids=[f"{d}-p{p}-eo{e}-{o}-B{b}" for d, p, e, o, b, *_ in _cases()])
def test_trainer_step(dtype, plan, epiopt, opt, B, D, H, Cn):
    """One step of the persistent trainer with the term, two ways.

    * anchor = the starting master: d = 0 everywhere, so the step equals the step without the term
      bit for bit (master, shadow, moments, work copies).
    * anchor = master + a perturbation p and mu = 1 / lr (SGD): w' = w - lr (g + mu d) is w0 - lr g up
      to a few roundings, where lr g comes from the step without the term from the same state.  Adam:
      m' = (1 - b1) g' and v' = (1 - b2) g'^2 with g' = g + mu d, g from the step without the term.
      Every element of W1, b1, W2 and b2 is checked, so each optimizer site (weight-gradient tiles,
      bias CTA, flat phase) is."""
    fp8 = dtype == "fp8"
    if H == 640:
        assert expected_bm_w(D, H) == 128, "this shape is meant to run 128-row weight-gradient tiles"
    fx = sat_fixture(B, 1, seed=B + 3, D=D, H=H, C=Cn)        # exact bias column sums: launches repeat bit for bit
    w = fx.master.cuda()
    plain = _step(fx, fp8, opt, plan, epiopt, 0.0, None)
    same = _step(fx, fp8, opt, plan, epiopt, 0.7, w.clone())
    for k, t in plain.items():
        if isinstance(t, torch.Tensor):
            assert torch.equal(t, same[k]), f"d = 0 changed {k}"
    lr = LR[opt]
    mu = 1.0 / lr if opt == "sgd" else 3.0
    pert = torch.randn(w.shape, generator=torch.Generator().manual_seed(5)) * 0.01
    real = torch.zeros(w.shape, dtype=torch.bool)          # the parameters; the padding between them is never read
    for e in Run(fx, fp8, opt).spec.entries:
        real[e.offset:e.offset + e.numel] = True
    anchor = (w + torch.where(real, pert, 0.0).cuda()).contiguous()
    got = _step(fx, fp8, opt, plan, epiopt, mu, anchor)
    mu32 = float(np.float32(mu))
    d = (w - anchor).double()
    if opt == "sgd":
        lrg = (w - plain["master"]).double()                  # lr g, to two roundings of |w|
        want = anchor.double() - lrg + (1 - float(np.float32(lr)) * mu32) * d
        tol = 8 * 2.0 ** -24 * (w.double().abs() + anchor.double().abs() + lrg.abs()) + 1e-30
        err = (got["master"].double() - want).abs()
        assert bool((err <= tol).all()), f"max err {float(err.max())} at {int(err.argmax())}"
    else:
        b1, b2 = 0.9, 0.999
        g = plain["m"].double() / (1 - float(np.float32(b1)))  # the moments start at 0
        gq = g + mu32 * d
        m_want = (1 - float(np.float32(b1))) * gq
        err = (got["m"].double() - m_want).abs()
        tol = 1e-5 * (g.abs() + mu32 * d.abs()) + 1e-30
        assert bool((err <= tol).all()), f"m: max err {float(err.max())} at {int(err.argmax())}"
        v_want = (1 - float(np.float32(b2))) * gq * gq
        errv = (got["v"].double() - v_want).abs()
        tolv = 4e-5 * (1 - float(np.float32(b2))) * (g.abs() + mu32 * d.abs()) ** 2 + 1e-30
        assert bool((errv <= tolv).all()), f"v: max err {float(errv.max())}"
        # the weights: Adam's last line on the kernel's own (checked) moments, t = 1, within the bound of
        # test_optim_spec_host.adam_w_bound
        ref, tolw = adam_w_bound(w.cpu().numpy(), got["m"].cpu().numpy(), got["v"].cpu().numpy(), F32(lr),
                                 F32(b1), F32(b2), F32(1e-8), 1)
        wk = got["master"].double().cpu().numpy()
        okw = (np.abs(wk - ref) <= tolw) | (wk == ref)
        assert okw.all(), f"w: {int((~okw).sum())} outside the bound, first at {first_bad(okw)}"
    assert int(torch.count_nonzero(got["grad"])) == 0


REPLAY = [("bf16", 4, "sgd"), ("bf16", 4, "adam"), ("bf16", 0, "sgd"), ("bf16", 3, "adam"), ("fp8", 4, "adam")]


@pytest.mark.parametrize("dtype,plan,opt", REPLAY, ids=[f"{d}-p{p}-{o}" for d, p, o in REPLAY])
def test_trainer_steps_in_one_launch_match_single_step_replay(dtype, plan, opt):
    """8 steps in one launch with an anchor against 8 single-step launches with the same anchor, bit for
    bit (the saturated fixture makes the bias column sums exact in any order)."""
    fp8, B, S = dtype == "fp8", 128, 8
    fx = sat_fixture(B, S, seed=11)
    anchor = (fx.master + 0.01 * torch.randn(fx.master.shape, generator=torch.Generator().manual_seed(2))).cuda()
    one = _run(fx, fp8, opt, 0.5, anchor)
    one.launch(plan, 1, S)
    got = one.state()
    rep = _run(fx, fp8, opt, 0.5, anchor)
    for s in range(S):
        rep.step.fill_(s)
        rep.tr.step_dev_ptr = rep.step.data_ptr() if opt == "adam" else 0
        rep.launch(plan, 1, 1, row0=s * B)
    want = rep.state()
    for k in got:
        if k in ("loss", "correct") or (k == "h_dq" and plan == 4):
            continue
        assert torch.equal(got[k], want[k]), k


# ------------------------------------------------------------------------------ engines
def close(a, b, rel=1e-4):
    """Equal up to the last-bit differences of the float-atomic bias column sums, which make two
    launches on real data differ (the saturated trainer fixtures above are exact)."""
    return float((a.double() - b.double()).abs().max()) <= rel * float(b.double().abs().max())


def _fused(prox_mu, optimizer="sgd", graph=False, dtype="bf16", B=256, S=1024, lr=0.05):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    cfg = FLConfig.for_world(1, model="mlp", hidden=256, batch_size=B, samples_per_client=S, learning_rate=lr,
                             optimizer=optimizer, cuda_graph=graph, dtype=dtype, prox_mu=prox_mu, non_iid_alpha=0.1)
    return FusedEngine(cfg, femnist_like(1, S, seed=7, only=0, alpha=0.1)[0])


@pytest.mark.parametrize("optimizer", ["sgd", "adam"])
def test_fused_engine_rounds_anchor_at_the_rounds_global(optimizer):
    """Two solo rounds: each round's upload is what a standalone FlatMLP computes from the same state
    with the anchor = the global model that round started from (genesis, then round 1's result), bit for
    bit; the host ledger re-executes both rounds with no mismatch."""
    eng = _fused(0.2, optimizer)
    o, P = eng.layout.offsets, eng.n_params
    genesis = eng.global_master.clone()
    for rnd in range(2):
        start = eng.global_master.clone()
        assert torch.equal(eng.work_master, start)
        m0 = (eng.trainer.m.clone(), eng.trainer.v.clone()) if optimizer == "adam" else None
        if rnd == 0:
            eng.capture()
        else:
            eng.run_round()
        torch.cuda.synchronize()
        # the Adam step base the round ran with (the plan's step word keeps it until the next round)
        step0 = eng.plan_bytes[eng.sz["plan_opt_step_off"]:eng.sz["plan_opt_step_off"] + 4].clone()
        up = eng.heap.view(o[f"upload_master{rnd & 1}"], [P], torch.float32).clone()
        from bflc_demo_b200.models.mlp import FlatMLP
        master = start.clone()
        step_word = step0.view(torch.int32).clone()
        ref = FlatMLP(eng.spec, master, master.bfloat16(), torch.zeros_like(master), eng.cfg.batch_size,
                      optimizer=optimizer, lr=eng.cfg.learning_rate, step_dev_ptr=step_word.data_ptr(),
                      prox_mu=0.2, anchor=start.clone())
        if m0 is not None:
            ref.m.copy_(m0[0])
            ref.v.copy_(m0[1])
        bar = torch.zeros(1, device="cuda", dtype=torch.int32)
        ref.train_epoch_fused(eng.x_bf, eng.y, eng.steps, bar.data_ptr())
        torch.cuda.synchronize()
        assert close(master, up), f"round {rnd}: upload differs from the standalone trainer"
        if rnd == 1:      # anchored at genesis instead, the same round ends measurably elsewhere
            master2 = start.clone()
            wrong = FlatMLP(eng.spec, master2, master2.bfloat16(), torch.zeros_like(master2), eng.cfg.batch_size,
                            optimizer=optimizer, lr=eng.cfg.learning_rate, step_dev_ptr=step_word.data_ptr(),
                            prox_mu=0.2, anchor=genesis)
            if m0 is not None:
                wrong.m.copy_(m0[0])
                wrong.v.copy_(m0[1])
            bar.zero_()
            wrong.train_epoch_fused(eng.x_bf, eng.y, eng.steps, bar.data_ptr())
            torch.cuda.synchronize()
            assert not close(master2, up, rel=1e-3)
        assert not torch.equal(eng.global_master, start)
    assert eng.drain_blocks() == []


def test_fused_engine_graph_replay_equals_eager():
    eager, graph = _fused(0.1, "adam", graph=False), _fused(0.1, "adam", graph=True)
    for e in (eager, graph):
        e.capture()
        for _ in range(3):
            e.run_round()
        torch.cuda.synchronize()
        assert e.drain_blocks() == []
    assert close(eager.global_master, graph.global_master)


def test_fused_engine_fp8_runs_with_prox():
    e = _fused(0.05, "adam", graph=True, dtype="fp8", B=256, S=1024)
    e.capture()
    for _ in range(2):
        st = e.run_round_e2e()
    assert st["epoch"] == 3 and e.drain_blocks() == []


def test_generic_engine_lenet_captured_equals_eager():
    """GenericFedEngine with FedProx and a recipe (decay, clipping): the captured training pass equals the
    eager one, and the term is in effect (mu = 0 ends elsewhere).  SGD: the convolutions' split-K float
    atomics make two runs differ in the last bits, and Adam would turn those differences on near-zero
    gradients into whole lr-sized steps; under SGD they stay at the size of the gradient noise, far below
    what the term moves."""
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import cifar_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import LeNet5
    out = {}
    for key, mu, graph in (("eager", 0.3, False), ("graph", 0.3, True), ("plain", 0.0, False)):
        cfg = FLConfig.for_world(1, batch_size=64, samples_per_client=256, learning_rate=0.05, model="lenet5",
                                 dataset="cifar10", optimizer="sgd", cuda_graph=graph, prox_mu=mu,
                                 weight_decay=0.01, clip_grad_norm=1.0)
        eng = GenericFedEngine(cfg, LeNet5(10), cifar_like(1, 256, seed=2, alpha=0.5)[0], rank=0, world=1, device=0)
        assert eng.recipe_step is not None and eng.recipe_step.prox_mu == mu
        eng.capture()
        for _ in range(2):
            eng.run_round()
        torch.cuda.synchronize()
        assert eng.drain_blocks() == []
        out[key] = eng.global_master.clone()
    gap = float((out["eager"] - out["graph"]).abs().max())
    moved = float((out["eager"] - out["plain"]).abs().max())
    assert close(out["eager"], out["graph"], rel=1e-4), gap
    assert moved > 20 * gap and not close(out["eager"], out["plain"], rel=1e-3), (moved, gap)


def test_generic_engine_prox_without_recipe_uses_the_recipe_kernel():
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import cifar_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import LeNet5
    cfg = FLConfig.for_world(1, batch_size=64, samples_per_client=128, learning_rate=0.05, model="lenet5",
                             dataset="cifar10", cuda_graph=False, prox_mu=0.2)
    eng = GenericFedEngine(cfg, LeNet5(10), cifar_like(1, 128, seed=2)[0], rank=0, world=1, device=0)
    assert eng.recipe_step is not None and eng.recipe_step.anchor is eng.global_master
    eng.capture()
    assert eng.drain_blocks() == []


def test_checkpoint_resume_continues_identically(tmp_path):
    from bflc_demo_b200.utils.checkpoint import load_checkpoint, save_checkpoint
    a = _fused(0.2, "adam")
    a.capture()
    a.run_round()
    torch.cuda.synchronize()
    save_checkpoint(str(tmp_path / "ck"), a)
    b = _fused(0.2, "adam")
    load_checkpoint(str(tmp_path / "ck"), b)
    b.capture()
    a.run_round()
    torch.cuda.synchronize()
    assert close(a.global_master, b.global_master)


def test_nccl_baseline_rejects_prox():
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.nccl_baseline import NcclBaselineEngine
    cfg = FLConfig.for_world(1, model="mlp", batch_size=128, samples_per_client=256, prox_mu=0.1)
    with pytest.raises(ValueError, match="FedProx"):
        NcclBaselineEngine(cfg, femnist_like(1, 256, seed=1, only=0)[0])
