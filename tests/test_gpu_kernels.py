"""Numerics of every hand-written sm_90a kernel against a plain PyTorch fp32 reference of the
same op.  Needs an H100 (``pytest -m gpu``); the native extension must be the code that runs --
``_native.C()`` raises if ``_C.so`` is missing, there is no eager fallback."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel(x, ref):
    return ((x.float() - ref.float()).norm() / (ref.float().norm() + 1e-12)).item()


def mk(*shape, dev="cuda"):
    c = shape[-1]
    cp = (c + 7) // 8 * 8
    t = (torch.randn(*shape[:-1], cp, device=dev) * 0.5).to(torch.bfloat16)
    return t[..., :c] if cp != c else t


@pytest.fixture(scope="module")
def G():
    from bflc_demo_b200.ops import gemm
    return gemm


@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (256, 256, 512), (200, 62, 784), (1000, 300, 1000)])
def test_gemm_kmajor(G, M, N, K):
    torch.manual_seed(0)
    a, b = mk(M, K), mk(N, K)
    d = G.gemm(a, b, out_dtype=torch.float32)
    assert rel(d, a.float() @ b.float().t()) < 1e-5


@pytest.mark.parametrize("M,N,K", [(256, 256, 512), (200, 256, 62), (130, 784, 300)])
def test_gemm_b_mn_major(G, M, N, K):
    torch.manual_seed(1)
    a, b = mk(M, K), mk(K, N)
    d = G.gemm(a, b, b_mn=True, out_dtype=torch.float32)
    assert rel(d, a.float() @ b.float()) < 1e-5


@pytest.mark.parametrize("M,N,K", [(256, 256, 512), (62, 256, 1000), (256, 784, 512)])
def test_gemm_both_mn_major(G, M, N, K):
    torch.manual_seed(2)
    a, b = mk(K, M), mk(K, N)
    d = G.gemm(a, b, a_mn=True, b_mn=True, out_dtype=torch.float32)
    assert rel(d, a.float().t() @ b.float()) < 1e-5


def test_gemm_fp8(G):
    torch.manual_seed(3)
    a = (torch.randn(256, 512, device="cuda") * 0.5).to(torch.float8_e4m3fn)
    b = (torch.randn(320, 512, device="cuda") * 0.5).to(torch.float8_e4m3fn)
    d = G.gemm(a, b, out_dtype=torch.float32)
    assert rel(d, a.float() @ b.float().t()) < 1e-5


def test_gemm_epilogues(G):
    torch.manual_seed(4)
    M, N, K = 300, 200, 784
    a, b = mk(M, K), mk(N, K)
    bias = torch.randn(N, device="cuda")
    colsum = torch.zeros(N, device="cuda")
    d = G.gemm(a, b, bias=bias, act=G.ACT_RELU, colsum=colsum)
    ref = torch.relu(a.float() @ b.float().t() + bias)
    assert rel(d, ref) < 4e-3 and rel(colsum, ref.sum(0)) < 1e-5
    assert rel(G.gemm(a, b, split_k=4), a.float() @ b.float().t()) < 1e-5
    mask = mk(M, N)
    d3 = G.gemm(a, b, aux_in=mask, act_bwd=1, out_dtype=torch.float32)
    assert rel(d3, (a.float() @ b.float().t()) * (mask.float() > 0)) < 1e-5
    pre = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    d4 = G.gemm(a, b, bias=bias, act=G.ACT_GELU, aux_out=pre, out_dtype=torch.float32)
    z = a.float() @ b.float().t() + bias
    assert rel(pre, z) < 4e-3 and rel(d4, torch.nn.functional.gelu(z)) < 1e-4
    d5 = G.gemm(a, b, aux_in=pre, act_bwd=2, out_dtype=torch.float32)
    zz = pre.float().requires_grad_(True)
    torch.nn.functional.gelu(zz).sum().backward()
    assert rel(d5, (a.float() @ b.float().t()) * zz.grad) < 1e-3
    ab, bb = mk(3, 130, 64), mk(3, 70, 64)
    assert rel(G.gemm(ab, bb, out_dtype=torch.float32), torch.bmm(ab.float(), bb.float().transpose(1, 2))) < 1e-5


def test_gemm_xent_and_accuracy(G):
    torch.manual_seed(5)
    M, N, K = 500, 62, 256
    a, b = mk(M, K), mk(N, K)
    bias = torch.randn(N, device="cuda") * 0.1
    labels = torch.randint(0, N, (M,), device="cuda", dtype=torch.int32)
    dl = torch.full((M, 64), 7.0, device="cuda", dtype=torch.bfloat16)
    loss = torch.zeros(1, device="cuda")
    corr = torch.zeros(1, device="cuda", dtype=torch.int32)
    colsum = torch.zeros(N, device="cuda")
    G.gemm_xent(a, b, labels, n_classes=N, bias=bias, dlogits=dl, grad_scale=1.0 / M,
                loss_sum=loss, correct=corr, colsum=colsum)
    logits = a.float() @ b.float().t() + bias
    ref_loss = torch.nn.functional.cross_entropy(logits, labels.long(), reduction="sum")
    p = torch.softmax(logits, 1)
    p[torch.arange(M), labels.long()] -= 1
    p /= M
    assert abs(loss.item() - ref_loss.item()) / abs(ref_loss.item()) < 1e-4
    assert rel(dl[:, :N], p) < 4e-3 and bool((dl[:, N:] == 0).all())
    assert int(corr.item()) == int((logits.argmax(1) == labels).sum().item())
    assert rel(colsum, p.sum(0)) < 1e-4
    corr2 = torch.zeros(2, device="cuda", dtype=torch.int32)
    G.gemm_argmax_acc(a, b, labels, corr2, n_classes=N, bias=bias)
    assert int(corr2[0].item()) == int(corr.item())


def test_mlp_training_step_matches_torch():
    """Six-kernel fused step (models/mlp.py) vs fp32 autograd of the same MLP."""
    from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec, torch_reference_step
    torch.manual_seed(6)
    spec = mlp_spec(784, 256, 62)
    master = torch.empty(spec.total)
    spec.init_(master, seed=1)
    master = master.cuda()
    # keep the master bf16-representable so both paths see the same weights
    master = master.bfloat16().float()
    shadow = master.bfloat16()
    grad = torch.zeros_like(master)
    B = 256
    tr = FlatMLP(spec, master, shadow, grad, B, lr=0.1)
    x = torch.rand(B, 784, device="cuda").bfloat16()
    y = torch.randint(0, 62, (B,), device="cuda", dtype=torch.int32)
    params = {k: v.clone() for k, v in spec.views(master).items()}
    loss_ref, new_ref, grads_ref = torch_reference_step(params, x, y, 0.1)
    tr.forward_backward(x, y)
    g = spec.views(grad)
    for k in ("w1", "b1", "w2", "b2"):
        assert rel(g[k], grads_ref[k]) < 2e-2, k
    assert abs(tr.loss_sum.item() / B - loss_ref.item()) < 2e-3
    tr.optimizer_step(1)
    for k, v in spec.views(master).items():
        assert rel(v, new_ref[k]) < 3e-3, k
    assert bool((grad == 0).all())


@pytest.mark.parametrize("plan,epiopt", [(-1, -1), (0, 0), (0, 1), (3, 0), (3, 1)])
@pytest.mark.parametrize("B,steps,opt", [(256, 3, "sgd"), (512, 4, "adam"), (200, 2, "sgd")])
def test_persistent_round_kernel_matches_six_kernel_path(B, steps, opt, plan, epiopt):
    """mlp_round_sm100.cu (one launch, grid barriers) vs the per-GEMM launches (models/mlp.py),
    for every phase plan: separate phases (0), whole chain per M-tile (1), fwd1 + 4-way sliced
    xent/dh chain (3); optimizer as a flat phase (epiopt 0) or inside the weight-gradient
    epilogues (1).  Compared on parameter DELTAS (a step moves a weight by O(1e-2) of its norm,
    so a weight-level tolerance would pass a badly scaled gradient), against the per-GEMM path
    AND against fp32 autograd of the same steps."""
    from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec
    torch.manual_seed(11)
    spec = mlp_spec(784, 256, 62)
    init = torch.empty(spec.total)
    spec.init_(init, seed=2)
    X = torch.rand(B * steps, 784, device="cuda").bfloat16()
    Y = torch.randint(0, 62, (B * steps,), device="cuda", dtype=torch.int32)
    outs = []
    for fused in (False, True):
        master = init.cuda().clone()
        shadow = master.bfloat16()
        grad = torch.zeros_like(master)
        tr = FlatMLP(spec, master, shadow, grad, B, lr=0.05 if opt == "sgd" else 1e-3, optimizer=opt)
        if fused:
            assert tr.fused_ok(steps)
            bar = torch.zeros(1, device="cuda", dtype=torch.int32)
            tr.train_epoch_fused(X, Y, steps, bar.data_ptr(), None, plan, epiopt)
        else:
            tr.train_epoch(X, Y, steps)
        torch.cuda.synchronize()
        outs.append((master.clone(), shadow.clone(), tr.loss_sum.item(), int(tr.correct.item()),
                     float(grad.abs().max())))
    (m0, s0, l0, c0, g0), (m1, s1, l1, c1, g1) = outs
    assert g0 == 0 and g1 == 0                       # both leave the gradient buffer zeroed
    assert abs(l0 - l1) / abs(l0) < 2e-3
    assert abs(c0 - c1) <= max(2, 0.01 * B * steps)
    w_init = spec.views(init.cuda())
    v0, v1 = spec.views(m0), spec.views(m1)
    tol = 2e-2 if opt == "sgd" else 0.1      # Adam's first steps are sign-like: noise-level grads flip
    for k in ("w1", "b1", "w2", "b2"):
        assert rel(v1[k] - w_init[k], v0[k] - w_init[k]) < tol, k
    assert rel(s1.float(), s0.float()) < 5e-3
    if opt == "sgd":
        # fp32 autograd of the same mini-batch steps (bf16 operands are the only difference)
        p = {k: v.clone().float() for k, v in w_init.items()}
        for i in range(steps):
            xb, yb = X[i * B:(i + 1) * B].float(), Y[i * B:(i + 1) * B].long()
            q = {k: v.clone().requires_grad_(True) for k, v in p.items()}
            loss = torch.nn.functional.cross_entropy(
                torch.relu(xb @ q["w1"].t() + q["b1"]) @ q["w2"].t() + q["b2"], yb)
            gr = torch.autograd.grad(loss, [q[k] for k in ("w1", "b1", "w2", "b2")])
            p = {k: (q[k] - 0.05 * g).detach() for k, g in zip(("w1", "b1", "w2", "b2"), gr)}
        for k in ("w1", "b1", "w2", "b2"):
            assert rel(v1[k] - w_init[k], p[k] - w_init[k]) < 6e-2, (k, rel(v1[k] - w_init[k], p[k] - w_init[k]))


@pytest.mark.parametrize("M,N,K", [(256, 256, 512), (512, 768, 1024), (300, 500, 200)])
def test_gemm_2cta(G, M, N, K):
    """CTA-pair kernel (2-CTA clusters, B multicast) against fp32 PyTorch."""
    torch.manual_seed(9)
    a, b = mk(M, K), mk(N, K)
    bias = torch.randn(N, device="cuda")
    d = G.gemm_2cta(a, b, out_dtype=torch.float32)
    assert rel(d, a.float() @ b.float().t()) < 1e-5
    d2 = G.gemm_2cta(a, b, bias=bias, act=G.ACT_RELU)
    assert rel(d2, torch.relu(a.float() @ b.float().t() + bias)) < 4e-3
