"""Phase plan 4 of the persistent MLP trainer (csrc/kernels/mlp_round_sm100.cu): fwd1 and the
fwd2 -> softmax-xent -> dh chain of an M-tile run in one 4-CTA cluster, and h reaches fwd2 through
distributed shared memory instead of global memory, a grid barrier and a TMA reload.

Plan 3 multiplies the same operands in the same K order, so after one step everything that does
not go through a float atomic is bit-identical: h, dlogits, dh, the weight masters, shadows, Adam
moments and (fp8) the MXFP8 work copies.  The biases and the loss are column / row sums by float
atomics, whose order differs between runs.  Over several steps those rounding differences feed back
into the forward pass, so multi-step runs are compared on parameter deltas as in
test_gpu_kernels.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel(x, ref):
    return ((x.float() - ref.float()).norm() / (ref.float().norm() + 1e-12)).item()


def _run(plan, dtype, opt, B, steps, hidden=256, dbg=None):
    from bflc_demo_b200._native import C
    from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec, sf_bytes
    torch.manual_seed(21)
    spec = mlp_spec(784, hidden, 62)
    init = torch.empty(spec.total)
    spec.init_(init, seed=4)
    xu8 = (torch.rand(B * steps, 784, device="cuda") ** 2 * 255).to(torch.uint8)
    y = torch.randint(0, 62, (B * steps,), device="cuda", dtype=torch.int32)
    xb = torch.empty(B * steps, 784, device="cuda", dtype=torch.bfloat16)
    xq = torch.zeros(B * steps, 784, device="cuda", dtype=torch.uint8)
    xsf = torch.full((sf_bytes(B * steps, 784),), 127, device="cuda", dtype=torch.uint8)
    C().prep_inputs(xu8, xb, xq, xsf, 1.0 / 255.0)
    master = init.cuda().clone()
    fp8 = dtype == "fp8"
    tr = FlatMLP(spec, master, master.bfloat16(), torch.zeros_like(master), B,
                 lr=(0.05 if opt == "sgd" else 1e-3), optimizer=opt, fp8=fp8)
    if fp8:
        tr.quantize_weights()
    bar = torch.zeros(1, device="cuda", dtype=torch.int32)
    tr.train_epoch_fused(xb, y, steps, bar.data_ptr(), dbg, plan, 1,
                         **({"x_q": xq, "x_sf": xsf} if fp8 else {}))
    torch.cuda.synchronize()
    out = {"init": init.cuda(), "master": master.clone(), "shadow": tr.shadow.clone(), "h": tr.h.clone(),
           "dlogits": tr.dlogits.clone(), "dh": tr.dh.clone(), "loss": tr.loss_sum.item(),
           "correct": int(tr.correct.item()), "grad_max": float(tr.grad.abs().max())}
    if opt == "adam":
        out["m"], out["v"] = tr.m.clone(), tr.v.clone()
    if fp8:
        out["work_q"], out["work_dq"] = tr.work_q.clone(), tr.work_dq.clone()
    return spec, out


ONE_STEP = ([(d, o, B) for d in ("bf16", "fp8") for o in ("sgd", "adam") for B in (128, 256, 512)]
            + [("bf16", o, 200) for o in ("sgd", "adam")])


@pytest.mark.parametrize("dtype,opt,B", ONE_STEP)
def test_plan4_one_step_matches_plan3(dtype, opt, B):
    spec, r3 = _run(3, dtype, opt, B, 1)
    _, r4 = _run(4, dtype, opt, B, 1)
    for k in ("h", "dlogits", "dh"):
        assert torch.equal(r4[k], r3[k]), k
    bufs = ("master", "shadow") + (("m", "v") if opt == "adam" else ())
    for buf in bufs:
        v3, v4 = spec.views(r3[buf]), spec.views(r4[buf])
        for k in ("w1", "w2"):
            assert torch.equal(v4[k], v3[k]), (buf, k)
    if dtype == "fp8":
        assert torch.equal(r4["work_q"], r3["work_q"])
        assert torch.equal(r4["work_dq"], r3["work_dq"])
    w0, v3, v4 = spec.views(r3["init"]), spec.views(r3["master"]), spec.views(r4["master"])
    for k in ("b1", "b2"):   # column sums by float atomics: equal up to summation order
        assert torch.allclose(v4[k] - w0[k], v3[k] - w0[k], rtol=1e-4, atol=1e-7), k
    assert abs(r4["loss"] - r3["loss"]) <= 1e-5 * abs(r3["loss"])
    assert r4["correct"] == r3["correct"]
    assert r4["grad_max"] == 0.0


MULTI_STEP = ([(d, o, 256, s) for d in ("bf16", "fp8") for o in ("sgd", "adam") for s in (4, 8)]
              + [("bf16", "sgd", 200, 4)])


@pytest.mark.parametrize("dtype,opt,B,steps", MULTI_STEP)
def test_plan4_steps_match_plan3(dtype, opt, B, steps):
    spec, r3 = _run(3, dtype, opt, B, steps)
    dbg = torch.zeros(steps, 32, device="cuda", dtype=torch.int64)
    _, r4 = _run(4, dtype, opt, B, steps, dbg=dbg)
    assert abs(r4["loss"] - r3["loss"]) / abs(r3["loss"]) < 2e-3
    assert abs(r4["correct"] - r3["correct"]) <= max(2, 0.01 * B * steps)
    w0, v3, v4 = spec.views(r3["init"]), spec.views(r3["master"]), spec.views(r4["master"])
    tol = 2e-2 if opt == "sgd" else 0.1
    for k in ("w1", "b1", "w2", "b2"):
        assert rel(v4[k] - w0[k], v3[k] - w0[k]) < tol, k
    assert rel(r4["shadow"], r3["shadow"]) < 5e-3
    # plan-4 stamps of CTA 0: fwd1 accumulator ready (16) <= h slice handed over (1) <= fwd1
    # epilogue done (17); whole h tile landed (6)
    d = dbg.cpu()
    for slot in (1, 6, 16, 17):
        assert bool((d[:, slot] > 0).all()), slot
    assert bool((d[:, 16] <= d[:, 1]).all()) and bool((d[:, 1] <= d[:, 17]).all())


def test_plan4_falls_back_to_plan0_without_hidden_256():
    spec, r0 = _run(0, "bf16", "sgd", 256, 1, hidden=128)
    _, r4 = _run(4, "bf16", "sgd", 256, 1, hidden=128)
    for k in ("h", "dlogits", "dh"):
        assert torch.equal(r4[k], r0[k]), k
    v0, v4 = spec.views(r0["master"]), spec.views(r4["master"])
    for k in ("w1", "w2"):
        assert torch.equal(v4[k], v0[k]), k
    w0 = spec.views(r0["init"])
    for k in ("b1", "b2"):
        assert torch.allclose(v4[k] - w0[k], v0[k] - w0[k], rtol=1e-4, atol=1e-7), k
    assert r4["correct"] == r0["correct"]
