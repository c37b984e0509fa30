"""Fine-tuning optimizer recipe on the GPU: the global-norm kernel against fp64, the recipe update
against torch's AdamW / SGD + LambdaLR + clip_grad_norm_, bit-identity of the no-op recipe with the
plain optimizer step, the schedule following the device step word inside a replayed graph, skipped
non-finite steps, and GenericFedEngine rounds (captured and eager, checkpoint resume)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def C():
    from bflc_demo_b200._native import C as _C
    return _C()


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _ws():
    return torch.zeros(C().grad_norm_workspace_bytes(), dtype=torch.uint8, device="cuda")


# ------------------------------------------------------------------------------ norm kernel
def _bert_base_params():
    from bflc_demo_b200.models.nets import BertBase
    return BertBase(2).spec.total


@pytest.mark.parametrize("n", [1, 3, 100003, "bert"])
def test_grad_norm_matches_fp64_and_is_bit_stable(n):
    n = _bert_base_params() if n == "bert" else n
    g = torch.Generator(device="cuda").manual_seed(n % 1000)
    grad = torch.randn(n, device="cuda", generator=g) * 1e-2
    ws, norms = _ws(), torch.zeros(4, device="cuda")
    C().grad_norm(grad, ws, norms, 0, 1.0)
    C().grad_norm(grad, ws, norms, 1, 1.0)
    torch.cuda.synchronize()
    ref = torch.linalg.vector_norm(grad.double())
    assert abs(float(norms[0]) - float(ref)) <= 1e-6 * float(ref)
    assert torch.equal(norms[0], norms[1])
    hdr = ws[:8].cpu()                          # GradNormState: coef, nonfinite
    coef, bad = hdr[:4].view(torch.float32).item(), hdr[4:8].view(torch.int32).item()
    assert coef == pytest.approx(min(1.0, 1.0 / (float(norms[0]) + 1e-6)), rel=1e-6) and bad == 0
    # graph replays: the ticket resets itself, the result does not move
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr, stream=s):
        C().grad_norm(grad, ws, norms, 2, 1.0)
    for k in range(3):
        norms[2] = -1
        gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(norms[2], norms[0]), k


def test_grad_norm_honours_predicate_and_validates():
    grad = torch.ones(1000, device="cuda")
    ws, norms = _ws(), torch.full((2,), -1.0, device="cuda")
    off = torch.zeros(1, dtype=torch.int32, device="cuda")
    C().grad_norm(grad, ws, norms, 0, 1.0, None, off.data_ptr())
    torch.cuda.synchronize()
    assert float(norms[0]) == -1.0
    with pytest.raises(RuntimeError):
        C().grad_norm(grad, ws, norms, 2, 1.0)                  # index outside norms
    with pytest.raises(RuntimeError):
        C().grad_norm(grad, ws[:16], norms, 0, 1.0)             # workspace too small
    with pytest.raises(RuntimeError):
        C().grad_norm(grad.double(), ws, norms, 0, 1.0)


# ------------------------------------------------------------------------------ update vs torch
def _spec():
    from bflc_demo_b200.models.flat import ParamSpec
    return ParamSpec([("w1", (64, 37)), ("b1", (64,)), ("ln_g", (13,)), ("emb", (50, 16)), ("b2", (5,)),
                      ("w2", (7, 9, 3)), ("bn_rvar", (21,))])


def _flat(spec, params):
    out = torch.zeros(spec.total, device="cuda")
    for e in spec.entries:
        out[e.offset:e.offset + e.numel] = params[e.name].detach().reshape(-1)
    return out


def _make_recipe(spec, steps, wd, sched, W, T, clip, n=None):
    from bflc_demo_b200.ops.optim import OptimRecipe, RecipeStep
    return RecipeStep(OptimRecipe(wd, sched, W, T, clip), spec, steps, "cuda", n=n)


@pytest.mark.parametrize("adam", [False, True])
@pytest.mark.parametrize("sched", ["constant", "linear", "cosine"])
@pytest.mark.parametrize("W", [0, 3])
@pytest.mark.parametrize("clip", [1.0, 100.0])
def test_recipe_matches_torch(adam, sched, W, clip):
    from bflc_demo_b200.ops.optim import lr_factor
    spec, steps, T, wd = _spec(), 20, 15, 0.1
    lr = 1e-2 if adam else 0.1
    gen = torch.Generator(device="cuda").manual_seed(11)
    w0 = torch.zeros(spec.total, device="cuda")
    for e in spec.entries:
        w0[e.offset:e.offset + e.numel] = torch.randn(e.numel, device="cuda", generator=gen) * 0.5
    grads = [torch.zeros(spec.total, device="cuda") for _ in range(steps)]
    for gk in grads:
        for e in spec.entries:
            gk[e.offset:e.offset + e.numel] = torch.randn(e.numel, device="cuda", generator=gen) * 0.1
    # torch reference: decay / no-decay groups, LambdaLR with the HF lambda, clip_grad_norm_
    views = spec.views(w0)
    params = {e.name: torch.nn.Parameter(views[e.name].clone()) for e in spec.entries}
    groups = [{"params": [params[e.name] for e in spec.entries if len(e.shape) >= 2], "weight_decay": wd},
              {"params": [params[e.name] for e in spec.entries if len(e.shape) == 1], "weight_decay": 0.0}]
    opt = (torch.optim.AdamW(groups, lr=lr, betas=(0.9, 0.999), eps=1e-8, foreach=False) if adam
           else torch.optim.SGD(groups, lr=lr, foreach=False))
    sch = torch.optim.lr_scheduler.LambdaLR(opt, lambda s: lr_factor(sched, s, W, T))
    # ours
    rs = _make_recipe(spec, steps, wd, sched, W, T, clip)
    master, grad = w0.clone(), torch.zeros(spec.total, device="cuda")
    shadow = master.to(torch.bfloat16)
    m = torch.zeros_like(master) if adam else None
    v = torch.zeros_like(master) if adam else None
    word = torch.zeros(1, dtype=torch.int32, device="cuda")
    triggered = 0
    for k in range(steps):
        gviews = spec.views(grads[k])
        for e in spec.entries:
            params[e.name].grad = gviews[e.name].clone()
        tn = float(torch.nn.utils.clip_grad_norm_(list(params.values()), clip))
        triggered += tn > clip
        opt.step()
        sch.step()
        grad.copy_(grads[k])
        rs(adam, master, grad, shadow, m, v, lr, k + 1, word.data_ptr(), k)
        torch.cuda.synchronize()
        ref = _flat(spec, params)
        assert rel(master, ref) < 1e-5, (k, rel(master, ref))
        assert torch.equal(shadow, master.to(torch.bfloat16)), k
        assert torch.count_nonzero(grad) == 0, k
        assert float(rs.norms[k]) == pytest.approx(tn, rel=1e-6), k
    assert (triggered == steps) if clip == 1.0 else (triggered == 0)
    assert int(rs.skipped) == 0


# ------------------------------------------------------------------------------ no-op recipe
@pytest.mark.parametrize("adam", [False, True])
@pytest.mark.parametrize("n", [1003, 40000])
def test_noop_recipe_is_bit_identical_to_optim_step(adam, n):
    from bflc_demo_b200.models.flat import ParamSpec
    from bflc_demo_b200.ops.optim import no_decay_mask
    spec = ParamSpec([("w", (n // 2,)), ("m", (2, n // 4))])      # 1-D and 2-D entries
    mask = no_decay_mask(spec, n).cuda()
    ws, norms = _ws(), torch.zeros(3, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(5)
    w0 = torch.randn(n, device="cuda", generator=gen)
    word = torch.full((1,), 7, dtype=torch.int32, device="cuda")
    outs = []
    for recipe in (False, True):
        master, shadow = w0.clone(), w0.to(torch.bfloat16)
        m = torch.zeros_like(master) if adam else None
        v = torch.zeros_like(master) if adam else None
        grad = torch.zeros(n, device="cuda")
        g2 = torch.Generator(device="cuda").manual_seed(6)
        for k in range(3):
            grad.copy_(torch.randn(n, device="cuda", generator=g2))
            if recipe:      # mask read, clip coefficient read (exactly 1), wd = 0, constant schedule
                C().grad_norm(grad, ws, norms, k, 1e30)
                C().optim_recipe_step(adam, master, grad, shadow, m, v, 1e-2, 0.9, 0.999, 1e-8, k + 1,
                                      word.data_ptr(), 0.0, mask, 0, 0, 0, ws)
            else:
                C().optim_step(adam, master, grad, shadow, m, v, 1e-2, 0.0, 0.9, 0.999, 1e-8, k + 1,
                               word.data_ptr(), 0, True)
        torch.cuda.synchronize()
        outs.append([t for t in (master, shadow, m, v, grad) if t is not None])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------ step word in a graph
def test_step_word_drives_the_schedule_inside_a_replayed_graph():
    spec = _spec()
    rs = _make_recipe(spec, 1, 0.1, "linear", 2, 10, 1.0)
    gen = torch.Generator(device="cuda").manual_seed(3)
    w0, g0 = torch.randn(spec.total, device="cuda", generator=gen), torch.randn(spec.total, device="cuda", generator=gen)
    master, grad, shadow = w0.clone(), g0.clone(), w0.to(torch.bfloat16)
    m, v = torch.zeros_like(w0), torch.zeros_like(w0)
    word = torch.zeros(1, dtype=torch.int32, device="cuda")

    def step():
        rs(True, master, grad, shadow, m, v, 1e-2, 1, word.data_ptr(), 0)

    step()                                                       # eager warm-up
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr, stream=s):
        step()

    def replay(w):
        word.fill_(w)
        master.copy_(w0); grad.copy_(g0); m.zero_(); v.zero_()  # noqa: E702
        gr.replay()
        torch.cuda.synchronize()
        return master.clone()

    first = replay(0)          # s = 0: warmup, lr_t = 0 -> AdamW leaves the weights
    assert torch.equal(first, w0)
    later = replay(4)          # s = 4: lr_t = lr * (10 - 4) / 8
    assert not torch.equal(later, first)
    assert torch.equal(replay(4), later)
    assert torch.equal(replay(0), first)


# ------------------------------------------------------------------------------ non-finite gradient
@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
def test_non_finite_gradient_skips_the_step(bad):
    spec = _spec()
    rs = _make_recipe(spec, 2, 0.1, "cosine", 0, 10, 1.0)
    gen = torch.Generator(device="cuda").manual_seed(4)
    master = torch.randn(spec.total, device="cuda", generator=gen)
    shadow = master.to(torch.bfloat16)
    m, v = torch.rand_like(master), torch.rand_like(master)
    word = torch.zeros(1, dtype=torch.int32, device="cuda")
    keep = [t.clone() for t in (master, shadow, m, v)]
    grad = torch.randn(spec.total, device="cuda", generator=gen)
    grad[spec.total // 3] = bad
    rs(True, master, grad, shadow, m, v, 1e-2, 1, word.data_ptr(), 0)
    torch.cuda.synchronize()
    for a, b in zip((master, shadow, m, v), keep):
        assert torch.equal(a, b)
    assert torch.count_nonzero(grad) == 0 and int(rs.skipped) == 1
    assert not math.isfinite(float(rs.norms[0]))
    grad.copy_(torch.randn(spec.total, device="cuda", generator=gen))     # the next good step runs
    rs(True, master, grad, shadow, m, v, 1e-2, 2, word.data_ptr(), 1)
    torch.cuda.synchronize()
    assert not torch.equal(master, keep[0]) and int(rs.skipped) == 1


def test_recipe_binding_validates():
    spec = _spec()
    n = spec.total
    w, g = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    mask = torch.zeros((n + 255) // 256, dtype=torch.int32, device="cuda")
    base = dict(adam=False, master=w, grad=g, shadow=None, m=None, v=None, lr=0.1, beta1=0.9, beta2=0.999,
                eps=1e-8, step=1, step_dev_ptr=0, decay=0.0, no_decay=None, schedule=0, warmup=0, total=0,
                clip_workspace=None)
    C().optim_recipe_step(**base)
    for bad in (dict(schedule=3), dict(schedule=1, warmup=5, total=5), dict(decay=0.1),
                dict(decay=0.1, no_decay=mask[:-1]), dict(adam=True), dict(grad=g[:-8]),
                dict(clip_workspace=torch.zeros(8, dtype=torch.uint8, device="cuda")), dict(warmup=-1)):
        with pytest.raises(RuntimeError):
            C().optim_recipe_step(**{**base, **bad})


# ------------------------------------------------------------------------------ engine
RECIPE = dict(weight_decay=0.01, lr_schedule="linear", warmup_steps=2, total_steps=40, clip_grad_norm=1.0)


def _engine(model, capture=True, **recipe):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import cifar_like, tokens_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import BertBase, ResNet18
    if model == "bert":
        cfg = FLConfig.for_world(1, model="bert", batch_size=8, samples_per_client=32, learning_rate=1e-3,
                                 optimizer="adam", cuda_graph=capture, **recipe)
        shard = tokens_like(1, 32, seed=3, seq_len=128)[0]
        net = BertBase(shard.n_classes, layers=2)
    else:
        cfg = FLConfig.for_world(1, model="resnet18", dataset="cifar10", batch_size=32, samples_per_client=128,
                                 learning_rate=0.05, cuda_graph=capture, **recipe)
        shard = cifar_like(1, 128, seed=2, alpha=0.0)[0]
        net = ResNet18(10)
    return GenericFedEngine(cfg, net, shard, rank=0, world=1, device=0)


# The models' backward passes accumulate some gradients with atomics, and bf16 activations turn a
# different summation order into differences of a few 1e-3 in a step's gradient norm.  While the
# weights move, each step feeds that difference into the next, and after a few steps two runs of the
# same training pass differ by percents.  So passes are compared with the weights held fixed (lr = 0,
# set before capture: the graph bakes the lr in), where a step's norm depends only on its batch, or at
# the first step of a pass, which starts from identical state.
def _save(eng):
    state = [t for t in (eng.work_master, eng.work_shadow, eng.grad, eng.m, eng.v, eng.skipped_steps, eng.plan_bytes)
             if t is not None]
    return state, [t.clone() for t in state]


def _restore(saved):
    for t, k in zip(*saved):
        t.copy_(k)


@pytest.mark.parametrize("model", ["bert", "resnet18"])
def test_engine_recipe_captured_rounds_learn(model):
    eng = _engine(model, True, **RECIPE)
    eng.capture()
    assert eng.graph_train is not None and not eng.capture_error
    losses, norms = [eng.read_state()["global_loss"]], [eng.grad_norms.clone()]
    for _ in range(4):
        eng.run_round()
        torch.cuda.synchronize()
        assert torch.isfinite(eng.grad_norms).all() and (eng.grad_norms > 0).all()
        norms.append(eng.grad_norms.clone())
        losses.append(eng.read_state()["global_loss"])
    assert int(eng.skipped_steps) == 0
    assert int(eng.opt_step_word) == 4 * eng.steps
    assert losses[-1] < losses[0], losses
    assert not torch.equal(norms[-1], norms[-2])
    assert eng.drain_blocks() == [] and eng.host_ledger.verify_chain()


@pytest.mark.parametrize("model", ["bert", "resnet18"])
def test_engine_recipe_graph_norms_match_eager(model):
    """The captured pass writes the same per-step norms as the pass run eagerly, from the same state
    and step word (weights held fixed, see the note above)."""
    eng = _engine(model, True, **RECIPE)
    eng.cfg.learning_rate = 0.0                  # FLConfig itself insists on lr > 0
    eng.capture()
    assert eng.graph_train is not None and not eng.capture_error
    eng.run_round()
    torch.cuda.synchronize()
    w0 = eng.work_master.clone()
    saved = _save(eng)
    with torch.cuda.stream(eng.stream):
        eng.local_training()
    eng.stream.synchronize()
    eager = eng.grad_norms.clone()
    # lr_t = 0: no update and no decay.  BatchNorm running statistics, which the training forward
    # itself updates in the flat buffer, are not the optimizer's.
    trained = torch.ones(eng.n_params, dtype=torch.bool, device="cuda")
    for e in eng.spec.entries:
        if e.name.endswith((".rmean", ".rvar")):
            trained[e.offset:e.offset + e.numel] = False
    assert torch.equal(eng.work_master[trained], w0[trained])
    _restore(saved)
    eng.grad_norms.fill_(float("nan"))
    with torch.cuda.stream(eng.stream):
        eng.graph_train.replay()
    eng.stream.synchronize()
    got = eng.grad_norms
    assert torch.isfinite(got).all() and (got > 0).all()
    assert torch.allclose(got, eager, rtol=2e-2, atol=0), (got, eager)
    assert int(eng.skipped_steps) == 0


@pytest.mark.parametrize("model", ["bert", "resnet18"])
def test_engine_recipe_checkpoint_resume_continues_the_schedule(model, tmp_path):
    from bflc_demo_b200.utils.checkpoint import load_checkpoint, save_checkpoint
    a = _engine(model, True, **RECIPE)
    a.capture()                                   # round 1 (eager) + capture
    a.run_round()                                 # round 2
    save_checkpoint(str(tmp_path / "ck.pt"), a)
    a.run_round()                                 # round 3
    torch.cuda.synchronize()
    b = _engine(model, True, **RECIPE)
    load_checkpoint(str(tmp_path / "ck.pt"), b)
    b.capture()                                   # its eager round is round 3
    torch.cuda.synchronize()
    assert int(b.opt_step_word) == int(a.opt_step_word) == 2 * a.steps
    assert torch.isfinite(b.grad_norms).all() and (b.grad_norms > 0).all()
    # round 3 starts from the saved global model on the same first batch
    assert torch.allclose(b.grad_norms[0], a.grad_norms[0], rtol=2e-2, atol=0), (a.grad_norms, b.grad_norms)


class _Calls:
    """Records the engine's calls into the native module, then forwards them."""

    def __init__(self, mod):
        self.mod, self.log = mod, []

    def __getattr__(self, name):
        f = getattr(self.mod, name)

        def call(*args):
            self.log.append((name, args))
            return f(*args)
        return call


def test_engine_default_config_keeps_the_plain_step():
    """With the default fields the training pass issues the plain optimizer step with the arguments it
    always had (the recipe kernel's no-op bit-identity is checked above, at the kernel)."""
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import cifar_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import LeNet5
    for recipe in ({}, dict(clip_grad_norm=1e30)):
        cfg = FLConfig.for_world(1, batch_size=64, samples_per_client=256, learning_rate=0.05, model="lenet5",
                                 dataset="cifar10", optimizer="adam", cuda_graph=False, **recipe)
        eng = GenericFedEngine(cfg, LeNet5(10), cifar_like(1, 256, seed=2, alpha=0.0)[0], rank=0, world=1, device=0)
        assert (eng.recipe_step is None) == (not recipe) and (eng.grad_norms is None) == (not recipe)
        eng.mod = _Calls(eng.mod)
        with torch.cuda.stream(eng.stream):
            saved = _save(eng)
            eng.local_training()
            _restore(saved)
        torch.cuda.synchronize()
        if recipe:          # the recipe steps go through ops/optim.py, not the plain entry point
            assert eng.mod.log == []
        else:
            want = [("optim_step", (True, eng.work_master, eng.grad, eng.work_shadow, eng.m, eng.v, 0.05, 0.0, 0.9,
                                    0.999, 1e-8, i + 1, eng.opt_step_ptr, 0, True)) for i in range(eng.steps)]
            assert len(eng.mod.log) == len(want)
            for (n1, a1), (n2, a2) in zip(eng.mod.log, want):
                assert n1 == n2 and len(a1) == len(a2)
                assert all((x is y) if isinstance(y, torch.Tensor) or y is None else x == y for x, y in zip(a1, a2))
        eng.mod = eng.mod.mod
        eng.capture()                                   # one eager round
        st = eng.read_state()
        assert st["epoch"] == 1 and math.isfinite(st["global_loss"])
