"""GroupNorm on the H100: the group-norm kernels (forward with ReLU and residual, backward with dx, the
residual gradient, dgamma and dbeta) against fp64 ``torch.nn.functional.group_norm``, bit-reproducible
and graph-capturable; the GroupNorm ResNet-18 end to end against an fp64 model; and generic-engine
rounds of it (graph replay, checkpoint / resume, the ledger, and the refusal of a batch-norm checkpoint)."""
import pytest
import torch
import torch.nn.functional as TF

from bflc_demo_b200._native import C
from bflc_demo_b200.ops import nn as F
from bflc_demo_b200.ops.nn import GN_EPS, GN_GROUPS

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
F64 = torch.float64
DEV = "cuda"


def _inputs(N, HW, Cc, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = (torch.randn(N, HW, HW, Cc, generator=g) * (0.5 + torch.rand(Cc, generator=g))
         + 2.0 * torch.randn(Cc, generator=g)).to(BF).to(DEV)
    gamma = (1.0 + 0.3 * torch.randn(Cc, generator=g)).to(DEV)
    beta = (0.2 * torch.randn(Cc, generator=g)).to(DEV)
    res = torch.randn(N, HW, HW, Cc, generator=g).to(BF).to(DEV)
    dy = torch.randn(N, HW, HW, Cc, generator=g).to(BF).to(DEV)
    return x, gamma, beta, res, dy


def _run(x, gamma, beta, res, dy, relu, acc=0.5):
    """The layer forward + backward through ops.nn.groupnorm; dgamma / dbeta start at ``acc`` (they
    accumulate)."""
    xk = x.clone().requires_grad_(True)
    rk = res.clone().requires_grad_(True) if res is not None else None
    gg = torch.full_like(gamma, acc)
    gb = torch.full_like(gamma, acc)
    y = F.groupnorm(xk, gamma, beta, gg, gb, relu=relu, residual=rk)
    y.backward(dy)
    torch.cuda.synchronize()
    return y.detach(), xk.grad, rk.grad if rk is not None else None, gg, gb


def _ref(x, gamma, beta, res, dy, mask):
    """fp64 group norm (+res) of the bf16 inputs; the backward takes dy masked by the kernel's own ReLU
    mask (``mask``: y > 0 of the kernel, or None)."""
    xt = x.double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    gt, bt = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    rt = res.double().permute(0, 3, 1, 2).contiguous().requires_grad_(True) if res is not None else None
    o = TF.group_norm(xt, GN_GROUPS, gt, bt, eps=GN_EPS)
    if rt is not None:
        o = o + rt
    g = dy.double().permute(0, 3, 1, 2)
    if mask is not None:
        g = g * mask.permute(0, 3, 1, 2)
    o.backward(g)
    nhwc = lambda t: t.permute(0, 2, 3, 1)   # noqa: E731
    return (nhwc(o.detach()), nhwc(xt.grad), nhwc(rt.grad) if rt is not None else None, gt.grad, bt.grad,
            nhwc(g), nhwc(xt.detach()))


@pytest.mark.parametrize("Cc, HW", [(64, 32), (128, 16), (256, 8), (512, 4), (64, 4), (512, 32)])
@pytest.mark.parametrize("relu, has_res", [(True, True), (True, False), (False, True), (False, False)])
def test_layer_against_fp64(Cc, HW, relu, has_res):
    N = 4
    x, gamma, beta, res, dy = _inputs(N, HW, Cc, seed=Cc * 7 + HW + 2 * relu + has_res)
    res = res if has_res else None
    y, dx, dres, gg, gb = _run(x, gamma, beta, res, dy, relu)
    mask = (y > 0).double() if relu else None
    o, rdx, rres, rdg, rdb, g, _ = _ref(x, gamma, beta, res, dy, mask)
    ry = o.clamp_min(0) if relu else o
    yd = y.double()
    # forward: fp32 arithmetic, then one bf16 rounding
    assert bool(((yd - ry).abs() <= 2.0 ** -8 * ry.abs() + 1e-3).all()), float((yd - ry).abs().max())
    # the residual gradient is the masked dy, exactly
    if has_res:
        assert torch.equal(dres.double(), g)
    # dx: fp32 group sums, one bf16 rounding
    scale = float(rdx.abs().max())
    err = (dx.double() - rdx).abs()
    assert bool((err <= 2.0 ** -8 * rdx.abs() + 1e-3 * scale).all()), float(err.max()) / scale
    # dgamma / dbeta accumulate onto 0.5; fp32 sums over N * HW^2 terms, bounded by the sums of |terms|
    xh = TF.group_norm(x.double().permute(0, 3, 1, 2), GN_GROUPS, eps=GN_EPS).permute(0, 2, 3, 1)
    tg = (g * xh).abs().sum((0, 1, 2))
    tb = g.abs().sum((0, 1, 2))
    assert bool(((gg.double() - 0.5 - rdg).abs() <= 1e-5 * tg + 1e-6).all()), float((gg.double() - 0.5 - rdg).abs().max())
    assert bool(((gb.double() - 0.5 - rdb).abs() <= 1e-5 * tb + 1e-6).all()), float((gb.double() - 0.5 - rdb).abs().max())


def test_bit_reproducible_and_examples_independent():
    x, gamma, beta, res, dy = _inputs(4, 16, 128, seed=11)
    a = _run(x, gamma, beta, res, dy, True)
    b = _run(x, gamma, beta, res, dy, True)
    for s, t in zip(a, b):
        assert torch.equal(s, t)
    # changing example 3 changes nothing of examples 0..2, bit for bit
    x2 = x.clone()
    x2[3] = x2[3] * 3 + 1
    c = _run(x2, gamma, beta, res, dy, True)
    assert torch.equal(c[0][:3], a[0][:3]) and torch.equal(c[1][:3], a[1][:3])
    assert not torch.equal(c[0][3], a[0][3])


def test_graph_replay_equals_eager():
    N, HW, Cc = 8, 8, 256
    x, gamma, beta, res, dy = _inputs(N, HW, Cc, seed=12)
    rows = N * HW * HW
    x2, r2, d2 = x.view(rows, Cc), res.view(rows, Cc), dy.view(rows, Cc)
    y, dx, dres = (torch.empty_like(x2) for _ in range(3))
    mean, rstd = (torch.empty(N * GN_GROUPS, device=DEV) for _ in range(2))
    gg, gb = torch.zeros(Cc, device=DEV), torch.zeros(Cc, device=DEV)
    pg, pb = torch.empty(N, Cc, device=DEV), torch.empty(N, Cc, device=DEV)

    def layer():
        gg.zero_()
        gb.zero_()
        C().groupnorm_fwd(x2, y, gamma, beta, mean, rstd, N, HW * HW, Cc, GN_GROUPS, GN_EPS, True, r2)
        C().groupnorm_bwd(d2, x2, y, gamma, mean, rstd, dx, gg, gb, dres, pg, pb, N, HW * HW, Cc, GN_GROUPS, True)

    layer()
    torch.cuda.synchronize()
    eager = [t.clone() for t in (y, dx, dres, gg, gb, pg, pb)]
    for t in (y, dx, dres, pg, pb):
        t.fill_(float("nan")) if t.dtype == torch.float32 else t.zero_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            layer()
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    for e, t in zip(eager, (y, dx, dres, gg, gb, pg, pb)):
        assert torch.equal(e, t)
    # each example's own dgamma / dbeta, summed in example order, are the parameter gradients
    sg, sb = torch.zeros_like(gg), torch.zeros_like(gb)
    for n in range(N):
        sg, sb = sg + pg[n], sb + pb[n]
    assert torch.equal(sg, gg) and torch.equal(sb, gb)
    for n in range(N):
        _, _, _, dgn, dbn, _, _ = _ref(x[n:n + 1], gamma, beta, res[n:n + 1], dy[n:n + 1],
                                       (y.view(x.shape)[n:n + 1] > 0).double())
        assert float((pg[n].double() - dgn).abs().max()) <= 1e-4 * float(dgn.abs().max()) + 1e-5
        assert float((pb[n].double() - dbn).abs().max()) <= 1e-4 * float(dbn.abs().max()) + 1e-5


def test_refuses_channels_not_a_multiple_of_the_groups():
    x = torch.zeros(1, 4, 4, 48, device=DEV, dtype=BF)
    g = torch.ones(48, device=DEV)
    with pytest.raises(ValueError, match="multiple of 32 groups"):
        F.groupnorm(x, g, g, None, None)
    with pytest.raises(RuntimeError, match="not a multiple of"):
        C().groupnorm_fwd(x.view(16, 48), x.view(16, 48), g, g, torch.empty(32, device=DEV),
                          torch.empty(32, device=DEV), 1, 16, 48, 32, GN_EPS, False, None)


# ------------------------------------------------------------------ GN ResNet-18 end to end
def _torch_weight(W, k, cin):
    cout = W.shape[0]
    return W[:, :k * k * cin].reshape(cout, k, k, cin).permute(0, 3, 1, 2)


def _resnet64(net, P, xb, y, q):
    """fp64 GN ResNet-18 on NCHW, from fp64 leaves P (torch layouts); ``q`` rounds each conv and norm
    output (identity: fp64; bf16: the emulation)."""
    def gn(name, t, relu, res=None):
        o = TF.group_norm(t, GN_GROUPS, P[f"{name}.gamma"], P[f"{name}.beta"], eps=GN_EPS)
        if res is not None:
            o = o + res
        return q(torch.relu(o) if relu else o)

    t = q(TF.conv2d(xb, P["stem.w"], padding=1))
    t = gn("stem.bn", t, True)
    for name, cin, c, stride, down in net.blocks:
        u = q(TF.conv2d(t, P[f"{name}.c1.w"], stride=stride, padding=1))
        u = gn(f"{name}.bn1", u, True)
        u = q(TF.conv2d(u, P[f"{name}.c2.w"], padding=1))
        idt = t
        if down:
            idt = gn(f"{name}.dbn", q(TF.conv2d(t, P[f"{name}.down.w"], stride=stride)), False)
        t = gn(f"{name}.bn2", u, True, res=idt)
    h = q(t.mean((2, 3)))
    return TF.cross_entropy(h @ P["fc.w"].t() + P["fc.b"], y)


def _leaves(net, master, shadow):
    Pm, Ps = net.spec.views(master), net.spec.views(shadow)
    P = {}
    for e in net.spec.entries:
        n = e.name
        if n == "stem.w":
            P[n] = _torch_weight(Ps[n].double(), 3, net.in_ch)
        elif n.endswith((".c1.w", ".c2.w")):
            P[n] = _torch_weight(Ps[n].double(), 3, Ps[n].shape[1] // 9)
        elif n.endswith(".down.w"):
            P[n] = _torch_weight(Ps[n].double(), 1, Ps[n].shape[1])
        elif n == "fc.w":
            P[n] = Ps[n].double()
        else:
            P[n] = Pm[n].double()
        P[n] = P[n].detach().clone().requires_grad_(True)
    return P


def _flat_grad(net, P):
    out = {}
    for e in net.spec.entries:
        g = P[e.name].grad
        if g.dim() == 4:
            g = g.permute(0, 2, 3, 1).reshape(g.shape[0], -1)
            g = TF.pad(g, (0, e.shape[1] - g.shape[1]))
        out[e.name] = g
    return out


@pytest.mark.parametrize("widths, N", [((64, 128, 256, 512), 4), ((32, 32, 64, 64), 8)])
def test_gn_resnet18_end_to_end_against_fp64(widths, N):
    from bflc_demo_b200.models.nets import ResNet18
    net = ResNet18(10, widths=widths, norm="group")
    master = torch.empty(net.spec.total, device=DEV)
    net.init_(master, seed=5)
    Pm = net.spec.views(master)
    gen = torch.Generator(device="cpu").manual_seed(6)
    for e in net.spec.entries:      # gamma / beta away from 1 / 0, so that a swapped pair shows
        if e.name.endswith(".gamma"):
            Pm[e.name].copy_(1.0 + 0.2 * torch.randn(e.shape, generator=gen))
        elif e.name.endswith(".beta") or e.name == "fc.b":
            Pm[e.name].copy_(0.1 * torch.randn(e.shape, generator=gen))
    shadow = master.to(BF)
    grad = torch.zeros_like(master)
    raw = torch.randint(0, 256, (N, 3, 32, 32), generator=gen, dtype=torch.uint8).to(DEV)
    y = torch.randint(0, 10, (N,), generator=gen).to(DEV)
    xb = net.preprocess(raw)
    loss = net.loss(net.bind(master, shadow, grad), xb, y.to(torch.int32))
    loss.backward()
    torch.cuda.synchronize()
    Gk = net.spec.views(grad)

    x64 = xb.double().permute(0, 3, 1, 2)
    res = {}
    for tag, q in (("fp64", lambda t: t), ("bf16", lambda t: t.to(BF).double())):
        P = _leaves(net, master, shadow)
        l64 = _resnet64(net, P, x64, y, q)
        l64.backward()
        res[tag] = (float(l64.detach()), _flat_grad(net, P))
    l_ref, g_ref = res["fp64"]
    l_emu, g_emu = res["bf16"]
    assert abs(float(loss) - l_ref) <= max(4 * abs(l_emu - l_ref), 2e-3 * abs(l_ref)), (float(loss), l_ref, l_emu)
    num = den = emu = 0.0
    for e in net.spec.entries:
        r, k, m = g_ref[e.name], Gk[e.name].double(), g_emu[e.name]
        num += float(((k - r) ** 2).sum())
        emu += float(((m - r) ** 2).sum())
        den += float((r ** 2).sum())
        rel, rel_emu = float((k - r).norm() / r.norm()), float((m - r).norm() / r.norm())
        assert rel <= max(4 * rel_emu, 5e-2), (e.name, rel, rel_emu)
    rel_all, emu_all = (num / den) ** 0.5, (emu / den) ** 0.5
    print(f"[gn resnet] widths {widths}: loss {float(loss):.6f} fp64 {l_ref:.6f} emu {l_emu:.6f}; "
          f"gradient rel err {rel_all:.3g} (bf16 emulation {emu_all:.3g})")
    assert rel_all <= max(4 * emu_all, 2e-2)


# ------------------------------------------------------------------ engine rounds
def _engine(norm, capture, shard, widths=(32, 32, 64, 64)):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import ResNet18
    cfg = FLConfig.for_world(1, model="resnet18", resnet_norm=norm, batch_size=16, samples_per_client=64,
                             learning_rate=0.005, cuda_graph=capture)
    eng = GenericFedEngine(cfg, ResNet18(10, widths=widths, norm=norm), shard, rank=0, world=1, device=0)
    if capture:
        eng.capture()
    return eng


def _rel(a, b, start):
    return float((a - b).norm() / (b - start).norm())


def test_gn_resnet_rounds_replay_resume_ledger_and_norm_refusal(tmp_path, monkeypatch):
    from bflc_demo_b200.data.synthetic import cifar_like
    from bflc_demo_b200.utils.checkpoint import load_checkpoint, save_checkpoint
    shard = cifar_like(1, 64, seed=3, alpha=0.0)[0]
    monkeypatch.setattr(F, "_split_k", lambda *a: 1)   # no split-K atomics in the weight gradients
    a = _engine("group", True, shard)        # capture: one eager round, then the graph
    assert a.capture_error == "" and a.graph_train is not None
    b = _engine("group", False, shard)
    c = _engine("group", False, shard)
    start = b.global_master.clone()
    for _ in range(2):
        a.run_round()
    for _ in range(3):
        b.run_round()
        c.run_round()
    torch.cuda.synchronize()
    # the head's bias sum still adds with fp32 atomics: when two eager runs agree bit for bit the replay
    # must too, otherwise it must sit within the eager runs' own spread
    spread = _rel(b.global_master, c.global_master, start)
    gap = _rel(a.global_master, b.global_master, start)
    print(f"[gn resnet engine] replay vs eager {gap:.3g}, eager vs eager {spread:.3g}")
    if spread == 0.0:
        assert torch.equal(a.global_master, b.global_master)
    assert gap <= max(4 * spread, 1e-3), (gap, spread)
    assert a.drain_blocks() == [] and b.drain_blocks() == [] and a.host_ledger.verify_chain()
    st = b.read_state()
    assert st["epoch"] == 3 and st["global_loss"] == st["global_loss"]
    acc = b.evaluate(shard)
    assert 0.0 <= acc <= 1.0

    path = str(tmp_path / "gn.pt")
    save_checkpoint(path, b)
    resumed = _engine("group", False, shard)
    load_checkpoint(path, resumed)
    assert torch.equal(resumed.global_master, b.global_master)
    mid = b.global_master.clone()
    b.run_round()
    resumed.run_round()
    torch.cuda.synchronize()
    if spread == 0.0:
        assert torch.equal(resumed.global_master, b.global_master)
    assert _rel(resumed.global_master, b.global_master, mid) <= max(4 * spread, 1e-3)
    assert resumed.drain_blocks() == [] and resumed.host_ledger.verify_chain()

    # a batch-norm run's checkpoint cannot be loaded by a group-norm engine, nor the other way round
    bn = _engine("batch", False, shard)
    bn.run_round()
    bpath = str(tmp_path / "bn.pt")
    save_checkpoint(bpath, bn)
    with pytest.raises(ValueError, match="n_params"):
        load_checkpoint(bpath, _engine("group", False, shard))
    with pytest.raises(ValueError, match="n_params"):
        load_checkpoint(path, _engine("batch", False, shard))
