"""NN kernels / autograd layer functions against PyTorch fp32 references, and the LeNet-5,
ResNet-18 and BERT model families end to end (loss goes down, gradients land in the flat
buffer, inference runs from an arbitrary weight buffer)."""
import pytest
import torch
import torch.nn.functional as TF

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def rel(x, ref):
    return ((x.float() - ref.float()).norm() / (ref.float().norm() + 1e-12)).item()


@pytest.fixture(scope="module")
def F():
    from bflc_demo_b200.ops import nn
    return nn


def _leaf(*shape, scale=0.5):
    return (torch.randn(*shape, device="cuda") * scale).to(BF).requires_grad_(True)


def test_linear_fwd_bwd(F):
    from bflc_demo_b200.ops import gemm as G
    torch.manual_seed(0)
    x = _leaf(300, 256)
    w = (torch.randn(120, 256, device="cuda") * 0.1).to(BF)
    b = torch.randn(120, device="cuda") * 0.1
    gw, gb = torch.zeros(120, 256, device="cuda"), torch.zeros(120, device="cuda")
    for act, ref_act in ((G.ACT_NONE, lambda t: t), (G.ACT_RELU, torch.relu), (G.ACT_GELU, TF.gelu)):
        gw.zero_(); gb.zero_(); x.grad = None
        y = F.linear(x, w, b, gw, gb, act)
        dy = torch.randn_like(y)
        y.backward(dy)
        xr = x.detach().float().requires_grad_(True)
        wr = w.float().requires_grad_(True)
        br = b.clone().requires_grad_(True)
        yr = ref_act(xr @ wr.t() + br)
        yr.backward(dy.float())
        assert rel(y, yr) < 1e-2
        assert rel(x.grad, xr.grad) < 2e-2 and rel(gw, wr.grad) < 2e-2 and rel(gb, br.grad) < 2e-2


@pytest.mark.parametrize("cin,cout,k,stride,pad,hw", [(3, 8, 5, 1, 0, 32), (16, 32, 3, 2, 1, 16),
                                                      (64, 64, 3, 1, 1, 8), (32, 64, 1, 2, 0, 8)])
def test_conv2d_fwd_bwd(F, cin, cout, k, stride, pad, hw):
    from bflc_demo_b200.ops import gemm as G
    torch.manual_seed(1)
    N = 4
    x = _leaf(N, hw, hw, cin)
    kc = k * k * cin
    kp = (kc + 7) // 8 * 8
    w = torch.zeros(cout, kp, device="cuda")
    w[:, :kc] = torch.randn(cout, kc, device="cuda") * 0.1
    w = w.to(BF)
    b = torch.randn(cout, device="cuda") * 0.1
    gw, gb = torch.zeros(cout, kp, device="cuda"), torch.zeros(cout, device="cuda")
    y = F.conv2d(x, w, b, gw, gb, k, k, stride, pad, G.ACT_RELU)
    dy = torch.randn_like(y)
    y.backward(dy)
    # reference: NCHW conv with the same weights ([cout, kh, kw, cin] -> [cout, cin, kh, kw])
    xr = x.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
    wr = w[:, :kc].float().view(cout, k, k, cin).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    br = b.clone().requires_grad_(True)
    yr = torch.relu(TF.conv2d(xr, wr, br, stride=stride, padding=pad))
    yr.backward(dy.float().permute(0, 3, 1, 2))
    assert rel(y, yr.permute(0, 2, 3, 1)) < 1e-2
    assert rel(x.grad, xr.grad.permute(0, 2, 3, 1)) < 3e-2
    assert rel(gw[:, :kc].view(cout, k, k, cin), wr.grad.permute(0, 2, 3, 1)) < 3e-2
    assert rel(gb, br.grad) < 3e-2


@pytest.mark.parametrize("n,cin,cout,k,stride,pad,hw", [
    (2, 64, 64, 3, 1, 1, 32),     # ResNet stage 1: one pixel tile = 4 image rows
    (3, 128, 128, 3, 1, 1, 16),   # 8-row tiles, 2 channel blocks per tap
    (4, 64, 128, 3, 2, 1, 32),    # strided: TMA elementStrides in forward / weight gradient
    (4, 64, 128, 1, 2, 0, 16),    # 1x1 strided downsample
    (5, 256, 64, 3, 1, 1, 4),     # tiny images: a pixel tile spans 8 images, 3 of them out of range
    (6, 64, 192, 3, 1, 1, 8),     # Cout not a multiple of the N tile
])
def test_conv2d_implicit_gemm(F, n, cin, cout, k, stride, pad, hw):
    """The implicit-GEMM path (tap-shifted 4-D TMA boxes, no im2col buffer) against fp32 cuDNN."""
    from bflc_demo_b200.ops import gemm as G
    torch.manual_seed(5)
    assert F.conv_is_implicit(hw, hw, cin, k, k, stride, pad, k * k * cin)
    x = _leaf(n, hw, hw, cin)
    kc = k * k * cin
    w = (torch.randn(cout, kc, device="cuda") * (1.0 / kc ** 0.5)).to(BF)
    b = torch.randn(cout, device="cuda") * 0.1
    gw, gb = torch.zeros(cout, kc, device="cuda"), torch.zeros(cout, device="cuda")
    y = F.conv2d(x, w, b, gw, gb, k, k, stride, pad, G.ACT_RELU)
    assert type(y.grad_fn).__name__.startswith("ConvImplicitFn")
    dy = torch.randn_like(y)
    y.backward(dy)
    xr = x.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
    wr = w.float().view(cout, k, k, cin).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    br = b.clone().requires_grad_(True)
    yr = torch.relu(TF.conv2d(xr, wr, br, stride=stride, padding=pad))
    yr.backward(dy.float().permute(0, 3, 1, 2))
    assert rel(y, yr.permute(0, 2, 3, 1)) < 1e-2
    assert rel(x.grad, xr.grad.permute(0, 2, 3, 1)) < 3e-2
    assert rel(gw.view(cout, k, k, cin), wr.grad.permute(0, 2, 3, 1)) < 3e-2
    assert rel(gb, br.grad) < 3e-2
    # second backward accumulates into gw (split-K atomics or += epilogue)
    g1 = gw.clone()
    x.grad = None
    y2 = F.conv2d(x, w, b, gw, gb, k, k, stride, pad, G.ACT_RELU)
    y2.backward(dy)
    assert rel(gw, 2 * g1) < 1e-2


def test_batchnorm_fwd_bwd(F):
    torch.manual_seed(2)
    x = _leaf(6, 8, 8, 32, scale=1.0)
    res = _leaf(6, 8, 8, 32)
    gamma = torch.rand(32, device="cuda") + 0.5
    beta = torch.randn(32, device="cuda") * 0.1
    gg, gb = torch.zeros(32, device="cuda"), torch.zeros(32, device="cuda")
    rm, rv = torch.zeros(32, device="cuda"), torch.ones(32, device="cuda")
    y = F.batchnorm(x, gamma, beta, gg, gb, rm, rv, True, True, res)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr = x.detach().float().requires_grad_(True)
    rr = res.detach().float().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    rm2, rv2 = torch.zeros(32, device="cuda"), torch.ones(32, device="cuda")
    yr = torch.relu(TF.batch_norm(xr.view(-1, 32), rm2, rv2, gr, br, True, 0.1, 1e-5).view_as(xr) + rr)
    yr.backward(dy.float())
    assert rel(y, yr) < 1e-2 and rel(x.grad, xr.grad) < 3e-2 and rel(res.grad, rr.grad) < 1e-2
    assert rel(gg, gr.grad) < 3e-2 and rel(gb, br.grad) < 3e-2
    assert rel(rm, rm2) < 1e-2 and rel(rv, rv2) < 1e-2
    # eval mode uses the running statistics
    ye = F.batchnorm(x.detach(), gamma, beta, None, None, rm, rv, False, False, None)
    yre = TF.batch_norm(x.detach().float().view(-1, 32), rm2, rv2, gamma, beta, False, 0.1, 1e-5)
    assert rel(ye.view(-1, 32), yre) < 1e-2


def test_layernorm_softmax_embedding_pool(F):
    from bflc_demo_b200._native import C
    torch.manual_seed(3)
    x = _leaf(200, 768, scale=1.0)
    gamma = torch.rand(768, device="cuda") + 0.5
    beta = torch.randn(768, device="cuda") * 0.1
    gg, gb = torch.zeros(768, device="cuda"), torch.zeros(768, device="cuda")
    y = F.layernorm(x, gamma, beta, gg, gb)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr = x.detach().float().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    yr = TF.layer_norm(xr, (768,), gr, br, 1e-12)
    yr.backward(dy.float())
    assert rel(y, yr) < 1e-2 and rel(x.grad, xr.grad) < 3e-2
    assert rel(gg, gr.grad) < 3e-2 and rel(gb, br.grad) < 3e-2
    # softmax rows
    s = (torch.randn(512, 128, device="cuda")).to(BF)
    p = torch.empty_like(s)
    C().softmax_fwd(s, p, 512, 128, 0.125)
    assert rel(p, torch.softmax(s.float() * 0.125, 1)) < 1e-2
    # embedding
    ids = torch.randint(0, 1000, (4 * 16,), device="cuda", dtype=torch.int32)
    table = (torch.randn(1000, 64, device="cuda")).to(BF)
    pos = (torch.randn(16, 64, device="cuda")).to(BF)
    gt, gp = torch.zeros(1000, 64, device="cuda"), torch.zeros(16, 64, device="cuda")
    e = F.embedding(ids, table, pos, gt, gp, 16)
    ref = table.float()[ids.long()] + pos.float().repeat(4, 1)
    assert rel(e, ref) < 1e-2
    de = torch.randn_like(e)
    e.backward(de)
    gt_ref = torch.zeros(1000, 64, device="cuda").index_add_(0, ids.long(), de.float())
    assert rel(gt, gt_ref) < 1e-3 and rel(gp, de.float().view(4, 16, 64).sum(0)) < 1e-3
    # pooling
    xi = _leaf(3, 8, 8, 16, scale=1.0)
    yp = F.maxpool2d(xi, 2, 2)
    dyp = torch.randn_like(yp)
    yp.backward(dyp)
    xr = xi.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
    ypr = TF.max_pool2d(xr, 2, 2)
    ypr.backward(dyp.float().permute(0, 3, 1, 2))
    assert rel(yp, ypr.permute(0, 2, 3, 1)) < 1e-3 and rel(xi.grad, xr.grad.permute(0, 2, 3, 1)) < 1e-2
    xa = _leaf(3, 4, 4, 16)
    ya = F.global_avgpool(xa)
    ya.backward(torch.ones_like(ya))
    assert rel(ya, xa.detach().float().mean((1, 2))) < 1e-2
    assert rel(xa.grad, torch.full_like(xa, 1 / 16).float()) < 1e-2


@pytest.mark.parametrize("fused,B,H", [(True, 2, 4), (True, 3, 12), (False, 2, 4)])
def test_attention_fwd_bwd(F, fused, B, H):
    """Fused one-kernel attention (attn_sm100.cu: QK^T -> softmax -> PV in registers / smem; backward
    with five wgmma GEMMs) and the unfused fallback, against fp32 PyTorch SDPA + autograd."""
    torch.manual_seed(4)
    S, D = 128, 64
    q, k, v = (_leaf(B * S, H * D, scale=0.7) for _ in range(3))
    o = F.attention(q, k, v, B, S, H, fused=fused)
    do = torch.randn_like(o)
    o.backward(do)

    def heads(t):
        return t.view(B, S, H, D).permute(0, 2, 1, 3)

    qr, kr, vr = (t.detach().float().requires_grad_(True) for t in (q, k, v))
    orf = TF.scaled_dot_product_attention(heads(qr), heads(kr), heads(vr))
    orf = orf.permute(0, 2, 1, 3).reshape(B * S, H * D)
    orf.backward(do.float())
    assert rel(o, orf) < 2e-2
    assert rel(q.grad, qr.grad) < 5e-2 and rel(k.grad, kr.grad) < 5e-2 and rel(v.grad, vr.grad) < 5e-2


def _train_steps(net, x, y, steps=6, lr=0.05):
    from bflc_demo_b200._native import C
    master = torch.empty(net.spec.total)
    net.init_(master, seed=1)
    master = master.cuda()
    shadow = master.to(BF)
    grad = torch.zeros_like(master)
    b = net.bind(master, shadow, grad)
    losses = []
    for _ in range(steps):
        loss = net.loss(b, x, y)
        loss.backward()
        losses.append(float(loss))
        assert float(grad.abs().sum()) > 0
        C().optim_step(False, master, grad, shadow, None, None, lr, 0.0, 0.9, 0.999, 1e-8, 1, 0, 0, True)
    return losses, master, shadow


def test_lenet5_trains_and_padding_stays_zero():
    from bflc_demo_b200.models.nets import LeNet5
    torch.manual_seed(5)
    net = LeNet5(10)
    xr = torch.randint(0, 255, (64, 3, 32, 32), device="cuda", dtype=torch.uint8)
    y = torch.randint(0, 10, (64,), device="cuda", dtype=torch.int32)
    losses, master, shadow = _train_steps(net, net.preprocess(xr), y, steps=8, lr=0.05)
    assert losses[-1] < losses[0]
    P = net.spec.views(master)
    assert float(P["conv1.w"][6:].abs().sum()) == 0 and float(P["fc.w"][:, 84:].abs().sum()) == 0
    cnt = net.correct(net.bind(master, shadow), net.preprocess(xr), y)
    assert 0 <= int(cnt) <= 64


def test_resnet18_trains():
    from bflc_demo_b200.models.nets import ResNet18
    torch.manual_seed(6)
    net = ResNet18(10)
    assert 11.0e6 < net.spec.total < 11.4e6
    xr = torch.randint(0, 255, (16, 3, 32, 32), device="cuda", dtype=torch.uint8)
    y = torch.randint(0, 10, (16,), device="cuda", dtype=torch.int32)
    losses, master, shadow = _train_steps(net, net.preprocess(xr), y, steps=5, lr=0.02)
    assert losses[-1] < losses[0]
    int(net.correct(net.bind(master, shadow), net.preprocess(xr), y))


def test_bert_small_trains():
    from bflc_demo_b200.models.nets import BertBase
    torch.manual_seed(7)
    net = BertBase(2, layers=2)
    ids = torch.randint(0, 30522, (8, 128), device="cuda")
    y = torch.randint(0, 2, (8,), device="cuda", dtype=torch.int32)
    losses, master, shadow = _train_steps(net, net.preprocess(ids), y, steps=5, lr=0.01)
    assert losses[-1] < losses[0]
    full = BertBase(2)
    assert 1.05e8 < full.spec.total < 1.15e8  # BERT-base parameter count


def test_mx8_forward_precision_linear_and_models(F):
    """Block-scaled fp8 forward (block-scaled e4m3 wgmma) behind ops.nn: the layer
    output tracks the bf16 layer, backward still produces bf16-path gradients, and the MLP /
    LeNet-5 configs BASELINE.json names as fp8 train."""
    from bflc_demo_b200.models.nets import LeNet5, MLPNet
    from bflc_demo_b200.ops import gemm as G
    torch.manual_seed(9)
    x = _leaf(256, 784)
    w = (torch.randn(256, 784, device="cuda") * 0.05).to(BF)
    b = torch.randn(256, device="cuda") * 0.1
    gw, gb = torch.zeros(256, 784, device="cuda"), torch.zeros(256, device="cuda")
    y_bf = F.linear(x, w, b, None, None, G.ACT_RELU).detach()
    prev = F.set_precision("mx8")
    try:
        assert prev == "bf16" and F.get_precision() == "mx8"
        y = F.linear(x, w, b, gw, gb, G.ACT_RELU)
        assert rel(y, y_bf) < 0.05
        y.backward(torch.randn_like(y))
        assert float(gw.abs().sum()) > 0 and x.grad is not None
        for net, xr, ncls in ((MLPNet(784, 256, 62), torch.randint(0, 255, (256, 784), device="cuda", dtype=torch.uint8), 62),
                              (LeNet5(10), torch.randint(0, 255, (64, 3, 32, 32), device="cuda", dtype=torch.uint8), 10)):
            yl = torch.randint(0, ncls, (xr.shape[0],), device="cuda", dtype=torch.int32)
            losses, master, shadow = _train_steps(net, net.preprocess(xr), yl, steps=8, lr=0.05)
            assert losses[-1] < losses[0]
    finally:
        F.set_precision("bf16")
