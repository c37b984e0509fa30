"""LoRA fine-tuning on the GPU: ``ops.nn.lora_linear`` against fp64 autograd, the frozen base, the
LoRA BERT / GPT models at genesis, and generic-engine rounds whose update is the adapter vector.
Needs an H100 (``pytest -m gpu``)."""
import pytest
import torch

from bflc_demo_b200.ops import gemm as G
from bflc_demo_b200.ops import nn as F

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
GPT_SMALL = dict(layers=2, hidden=128, heads=2, ffn=256, vocab=512, max_pos=128)


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _act64(z, act):
    if act == G.ACT_RELU:
        return z.clamp_min(0)
    if act == G.ACT_GELU:
        return torch.nn.functional.gelu(z)
    return z


@pytest.mark.parametrize("act", [G.ACT_NONE, G.ACT_RELU, G.ACT_GELU], ids=["none", "relu", "gelu"])
@pytest.mark.parametrize("r", [8, 16, 64])
@pytest.mark.parametrize("shape", [(256, 768, 768), (200, 3072, 768), (136, 768, 3072)],
                         ids=lambda s: "x".join(map(str, s)))
def test_lora_linear_against_fp64(act, r, shape):
    M, N, K = shape
    g = torch.Generator(device="cuda").manual_seed(M + N + r + act)
    x = (torch.randn(M, K, generator=g, device="cuda") * 0.5).to(BF)
    w = (torch.randn(N, K, generator=g, device="cuda") / K ** 0.5).to(BF)
    b = torch.randn(N, generator=g, device="cuda") * 0.1
    a = (torch.randn(r, K, generator=g, device="cuda") / K ** 0.5).to(BF)
    bl = (torch.randn(N, r, generator=g, device="cuda") * 0.1).to(BF)
    dy = torch.randn(M, N, generator=g, device="cuda").to(BF)
    scale = 2.0
    w0, b0 = w.clone(), b.clone()
    ga, gbl = torch.zeros(r, K, device="cuda"), torch.zeros(N, r, device="cuda")
    xg = x.clone().requires_grad_(True)
    y = F.lora_linear(xg, w, b, a, bl, ga, gbl, scale, act)
    y.backward(dy)
    torch.cuda.synchronize()
    # forward: u = scale * x a^T is rounded to bf16 before the tail, as the kernel path does
    u = G.gemm(x, a, alpha=scale).double()
    x64, w64, a64, bl64 = (t.double() for t in (x, w, a, bl))
    z = x64 @ w64.T + u @ bl64.T + b.double()
    assert rel(y, _act64(z, act)) < 8e-3
    # gradients against fp64 autograd of the same function, u's bf16 rounding modelled: its value is
    # the kernel path's u, its gradient that of scale * x a^T (a straight-through term)
    xr, ar, blr = (t.detach().clone().requires_grad_(True) for t in (x64, a64, bl64))
    s_xa = scale * (xr @ ar.T)
    yr = _act64(xr @ w64.T + (u + s_xa - s_xa.detach()) @ blr.T + b.double(), act)
    yr.backward(dy.double())
    assert rel(gbl, blr.grad) < 2e-2
    assert rel(ga, ar.grad) < 2e-2
    assert rel(xg.grad, xr.grad) < 2e-2
    # the frozen weight and bias are untouched
    assert torch.equal(w, w0) and torch.equal(b, b0)


def test_lora_linear_accumulates_and_refuses_mx8():
    M, N, K, r = 128, 256, 128, 8
    x = torch.randn(M, K, device="cuda").to(BF)
    w, b = torch.randn(N, K, device="cuda").to(BF), torch.zeros(N, device="cuda")
    a, bl = torch.randn(r, K, device="cuda").to(BF), torch.randn(N, r, device="cuda").to(BF)
    ga, gbl = torch.zeros(r, K, device="cuda"), torch.zeros(N, r, device="cuda")
    dy = torch.randn(M, N, device="cuda").to(BF)
    F.lora_linear(x, w, b, a, bl, ga, gbl, 1.0).backward(dy)
    ga1, gbl1 = ga.clone(), gbl.clone()
    F.lora_linear(x, w, b, a, bl, ga, gbl, 1.0).backward(dy)
    torch.cuda.synchronize()
    assert rel(ga, 2 * ga1) < 1e-5 and rel(gbl, 2 * gbl1) < 1e-5
    prev = F.set_precision("mx8")
    try:
        with pytest.raises(ValueError):
            F.lora_linear(x, w, b, a, bl, ga, gbl, 1.0)
    finally:
        F.set_precision(prev)
    with pytest.raises(ValueError):
        F.lora_linear(x, w, b, a[:, :64].contiguous(), bl, ga, gbl, 1.0)


def _models():
    from bflc_demo_b200.models.nets import GPT, BertBase
    return {
        "gpt": lambda: GPT(**GPT_SMALL),
        "bert_padded": lambda: BertBase(2, layers=2, pad_id=0),
        "bert_packed": lambda: BertBase(2, layers=2, pad_id=0, packed=True),
    }


def _ids(kind):
    torch.manual_seed(3)
    if kind == "gpt":
        ids = torch.randint(0, 512, (4, 128), device="cuda")
        return ids, torch.randint(0, 512, (4, 128), device="cuda", dtype=torch.int32)
    lens, S = [128, 100, 37, 5], 128
    ids = torch.zeros(len(lens), S, dtype=torch.int64, device="cuda")
    for i, n in enumerate(lens):
        ids[i, :n] = torch.randint(1, 30522, (n,), device="cuda")
    return ids, torch.tensor([0, 1, 1, 0], device="cuda", dtype=torch.int32)


@pytest.mark.parametrize("kind", list(_models()))
def test_lora_model_genesis_is_the_base_and_only_adapters_train(kind):
    from bflc_demo_b200.models.lora import LoRANet
    base = _models()[kind]()
    net = LoRANet(base, rank=8, alpha=16, targets="q,v,ff1")
    bm, bs = net.base_buffers("cuda")
    bm0 = bm.clone()
    master = torch.empty(net.spec.total, device="cuda")
    net.init_(master, seed=5)
    shadow, grad = master.to(BF), torch.zeros_like(master)
    lb = net.bind(master, shadow, grad)
    plain = base.bind(bm, bs, None)
    if kind != "gpt":                       # the base's head is the task head's stand-in here
        plain.P["cls.w"], plain.S["cls.w"] = lb.P["cls.w"], lb.S["cls.w"]
        plain.P["cls.b"], plain.S["cls.b"] = lb.P["cls.b"], lb.S["cls.b"]
    ids, y = _ids(kind)
    x = net.preprocess(ids)
    with torch.no_grad():
        h_lora = net.features(lb, x, False)
        h_base = base.features(plain, x, False)
    assert torch.equal(h_lora, h_base)
    loss = net.loss(lb, x, y)
    loss.backward()
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    assert torch.equal(bm, bm0)
    G_ = net.spec.views(grad)
    # B = 0 at genesis: dL/dA = 0 and dL/dB = dz^T u != 0 for every adapted projection
    for proj, (an, bn) in net.adapted.items():
        assert torch.count_nonzero(G_[an]) == 0, an
        assert float(G_[bn].abs().sum()) > 0, bn
    if kind != "gpt":
        assert float(G_["cls.w"].abs().sum()) > 0


def test_lora_gradients_reach_both_adapter_factors_once_b_is_nonzero():
    """With B != 0 (as after the first rounds) the backward reaches A as well as B in every
    adapted projection, through the whole model."""
    from bflc_demo_b200.models.lora import LoRANet
    from bflc_demo_b200.models.nets import GPT
    net = LoRANet(GPT(**GPT_SMALL), rank=16, targets="q,v")
    master = torch.empty(net.spec.total, device="cuda")
    net.init_(master, seed=2)
    P = net.spec.views(master)
    g = torch.Generator(device="cuda").manual_seed(9)
    for _, bn in net.adapted.values():
        P[bn].copy_(torch.randn(P[bn].shape, generator=g, device="cuda") * 0.05)
    shadow, grad = master.to(BF), torch.zeros_like(master)
    lb = net.bind(master, shadow, grad)
    ids, y = _ids("gpt")
    loss = net.loss(lb, net.preprocess(ids), y)
    loss.backward()
    torch.cuda.synchronize()
    Gv = net.spec.views(grad)
    for _, (an, bn) in net.adapted.items():
        assert torch.isfinite(Gv[an]).all() and float(Gv[an].abs().sum()) > 0
        assert torch.isfinite(Gv[bn]).all() and float(Gv[bn].abs().sum()) > 0


# --------------------------------------------------------------------------- engine rounds
def _engine(kind="gpt", rounds=0, lr=2e-3, capture=False, **cfg_kw):
    """A 1-GPU LoRA engine; lr 0 freezes the adapters too (set after the config's lr > 0 check)."""
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.lora import LoRANet
    if kind == "gpt":
        from bflc_demo_b200.data.synthetic import lm_corpus_like
        from bflc_demo_b200.models.nets import GPT
        cfg = FLConfig.for_world(1, model="gpt", batch_size=16, samples_per_client=64, learning_rate=lr or 1e-3,
                                 optimizer="adam", cuda_graph=capture, val_samples=32, lora_rank=8, **cfg_kw)
        shard = lm_corpus_like(1, 64, seed=3, seq_len=128, vocab=512, only=0)[0]
        base = GPT(**GPT_SMALL)
    else:
        from bflc_demo_b200.data.synthetic import tokens_like
        from bflc_demo_b200.models.nets import BertBase
        cfg = FLConfig.for_world(1, model="bert", batch_size=8, samples_per_client=16, learning_rate=lr or 1e-3,
                                 cuda_graph=capture, lora_rank=8, **cfg_kw)
        shard = tokens_like(1, 16, seed=3, seq_len=128, min_len=32)[0]
        base = BertBase(shard.n_classes, layers=2, pad_id=0)
    net = LoRANet(base, cfg.lora_rank, cfg.lora_alpha, cfg.lora_targets)
    eng = GenericFedEngine(cfg, net, shard, rank=0, world=1, device=0)
    eng.cfg.learning_rate = lr
    if capture:
        eng.capture()
    for _ in range(rounds):
        eng.run_round()
    return eng, net, shard


@pytest.mark.parametrize("kind", ["gpt", "bert"])
def test_lora_engine_rounds_train_the_adapters_only(kind):
    eng, net, shard = _engine(kind, rounds=3)
    torch.cuda.synchronize()
    assert eng.n_params == net.spec.total
    assert eng.drain_blocks() == [] and eng.host_ledger.verify_chain()
    bm, _ = net.base_buffers(eng.dev)
    fresh = torch.empty_like(bm)
    net.base.init_(fresh, seed=net.base_seed)
    assert torch.equal(bm, fresh)                         # the base never moved
    assert torch.isfinite(eng.global_master).all()
    B = net.spec.views(eng.global_master)
    assert any(float(B[bn].abs().sum()) > 0 for _, bn in net.adapted.values())


def test_lora_gpt_rounds_lower_the_loss_below_the_base():
    """Seeded LoRA rounds on a GPT base: the global model's loss on the fine-tuning shard falls
    below the base model's (the genesis LoRA model computes exactly the base)."""
    eng, net, shard = _engine("gpt", rounds=0, lr=3e-3)
    x, y = eng.x[:16], shard.y[:16].to(eng.dev, torch.int32)

    @torch.no_grad()
    def global_loss():
        b = net.bind(eng.global_master, eng.global_shadow, None)
        return float(net.loss(b, x, y))

    base = global_loss()
    for _ in range(6):
        eng.run_round()
    torch.cuda.synchronize()
    tuned = global_loss()
    print(f"LoRA GPT loss on the fine-tuning shard: base {base:.4f}, after 6 rounds {tuned:.4f}")
    assert eng.drain_blocks() == [] and eng.host_ledger.verify_chain()
    assert tuned < base, (base, tuned)


def test_lora_captured_round_equals_eager_at_lr0():
    eng, _, _ = _engine("gpt", lr=0.0, capture=True)
    assert eng.capture_error == "" and eng.graph_train is not None

    def one(eager):
        with torch.cuda.stream(eng.stream):
            eng.loss_sum.zero_()
            if eager:
                eng.local_training()
            else:
                eng.graph_train.replay()
        eng.stream.synchronize()
        return eng.loss_sum.clone()

    g, e = one(False), one(True)
    assert torch.isfinite(g).all() and torch.equal(g, e), (g, e)


@pytest.mark.parametrize("kw", [dict(server_opt="momentum"), dict(aggregation="median"),
                                dict(dp_clip=1.0, dp_noise=0.1), dict(prox_mu=0.01)],
                         ids=["fedavgm", "median", "dp", "fedprox"])
def test_lora_protocol_features_run_on_the_adapter_vector(kw):
    eng, net, _ = _engine("gpt", rounds=2, **kw)
    torch.cuda.synchronize()
    assert eng.n_params == net.spec.total
    assert eng.drain_blocks() == [] and eng.host_ledger.verify_chain()
    assert torch.isfinite(eng.global_master).all()


def test_lora_checkpoint_resume_and_base_digest_refusal(tmp_path):
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.lora import LoRANet
    from bflc_demo_b200.models.nets import GPT
    from bflc_demo_b200.utils.checkpoint import load_checkpoint, save_checkpoint
    eng, net, shard = _engine("gpt", rounds=2)
    path = str(tmp_path / "lora.pt")
    save_checkpoint(path, eng)
    cfg = eng.cfg
    same = GenericFedEngine(cfg, LoRANet(GPT(**GPT_SMALL), 8), shard, rank=0, world=1, device=0)
    load_checkpoint(path, same)
    assert torch.equal(same.global_master, eng.global_master)
    same.run_round()
    assert same.drain_blocks() == [] and same.host_ledger.verify_chain()
    assert same.read_state()["epoch"] == eng.read_state()["epoch"] + 1
    other = GenericFedEngine(cfg, LoRANet(GPT(**GPT_SMALL), 8, base_seed=77), shard, rank=0, world=1, device=0)
    with pytest.raises(ValueError, match="base"):
        load_checkpoint(path, other)


# ------------------------------------------------------------- end to end against fp64
def test_lora_gpt_loss_and_adapter_gradients_against_fp64():
    """The LoRA GPT (adapters on q, v, o and the GELU ff1, B != 0, scale 2) end to end: loss and every
    adapter gradient against an independent fp64 model (the GPT conformance suite's ``fp64_gpt`` with
    each adapted projection run through ``lora_linear64``), with a bf16 emulation of the kernels'
    storage points as the yardstick: ||kernel - fp64|| <= RATIO ||emulation - fp64|| + floor.  A
    misrouted adapter (q's on k, swapped layers, A and B exchanged), a wrong scale or a gradient bound
    to the wrong view is far outside that."""
    import math

    import test_gpu_gpt_conformance as GC
    import test_gpu_model_conformance as MC
    from test_lora_host import lora_linear64

    from bflc_demo_b200.models.lora import LoRANet
    base_net = GC.make()[0]
    net = LoRANet(base_net, rank=8, alpha=16, targets="q,v,o,ff1")
    bm = torch.empty(base_net.spec.total)
    base_net.init_(bm, seed=1)
    g = torch.Generator().manual_seed(10)
    for k, v in base_net.spec.views(bm).items():     # non-trivial biases and norms, as GC.make
        if k.endswith(".b") or k.endswith(".beta"):
            v.copy_(torch.randn(v.shape, generator=g) * 0.02)
        elif k.endswith(".gamma"):
            v.copy_(1 + torch.randn(v.shape, generator=g) * 0.05)
    net._base_cpu = bm
    master = torch.empty(net.spec.total)
    net.init_(master, seed=4)
    P = net.spec.views(master)
    for _, bn in net.adapted.values():
        P[bn].copy_(torch.randn(P[bn].shape, generator=g) * 0.05)
    master = master.cuda()
    shadow, grad = master.to(BF), torch.zeros_like(master)
    lb = net.bind(master, shadow, grad)
    ids, y = GC.data()
    loss = net.loss(lb, ids, y)
    loss.backward()
    torch.cuda.synchronize()
    bmc, bsc = net.base_buffers("cuda")

    def run64(emul):
        Pd = MC.fp64_params(base_net, bmc, bsc, "cuda")
        Sa = net.spec.views(shadow)
        ad = {n: Sa[n].detach().double().clone().requires_grad_(True) for e in net.adapted.values() for n in e}
        by_w = {id(Pd[f"{proj}.w"]): (ad[a], ad[b]) for proj, (a, b) in net.adapted.items()}
        m = MC.Model64(emul)
        plain = m.linear

        def linear(x, w, b, act=G.ACT_NONE):
            if id(w) not in by_w:
                return plain(x, w, b, act)
            A, B = by_w[id(w)]
            z = lora_linear64(x, w, b, A, B, net.scale, round_u=m.r)
            return m.r(z) if act == G.ACT_NONE else m.r(MC.gelu_ref(m.r(z)))

        m.linear = linear
        l64 = GC.fp64_gpt(base_net, Pd, ids, y, m)
        l64.backward()
        return l64.detach(), {k: v.grad for k, v in ad.items()}

    f64, emu = run64(False), run64(True)
    gv = net.spec.views(grad)
    items = [("loss", loss.detach().double().reshape(()), f64[0], emu[0])]
    items += [(n, gv[n].double(), f64[1][n], emu[1][n]) for e in net.adapted.values() for n in e]
    bad, report = [], []
    for name, k, ref, em in items:
        ek = float((k - ref.reshape(k.shape)).norm())
        ee = float((em.reshape(k.shape) - ref.reshape(k.shape)).norm())
        rn = float(ref.norm())
        floor = (GC.BF_U if k.numel() == 1 else 2.0 ** -16) * rn + 1e-30
        report.append(f"{name}: {ek / ee if ee else 0:.2f}")
        if not math.isfinite(ek) or ek > GC.RATIO * ee + floor:
            bad.append(f"{name}: ||kernel - fp64|| {ek:.3g} > {GC.RATIO} x ||emulation - fp64|| {ee:.3g} + {floor:.3g}")
    print("LoRA GPT e2e ratios:", ", ".join(report))
    assert not bad, "; ".join(bad)


def test_lora_committee_score_is_hits_over_targets_and_rounds_within_measured_spread():
    """Committee scores equal hits / targets of the bound candidate.  Trained rounds are compared only
    within a spread measured from repeated runs (the adapter weight gradients go through split-K fp32
    atomics, so runs are not assumed bit-reproducible): captured against eager within 4x the larger
    spread of two captured runs and of two eager runs.  Adam turns the atomics'
    last-bit differences in near-zero gradients into lr-sized steps, so the measured spread varies
    from run to run (about 1e-7 to 3e-4 after 4 rounds at lr 2e-3 on an H100)."""
    from bflc_demo_b200.engine.base import parse_block_record

    def captured():
        e, _, _ = _engine("gpt", capture=True, lr=2e-3)
        for _ in range(3):
            e.run_round()
        return e

    a, a2 = captured(), captured()
    b, _, _ = _engine("gpt", rounds=4)
    c, _, _ = _engine("gpt", rounds=4)
    torch.cuda.synchronize()
    d_eager = float((c.global_master - b.global_master).abs().max())
    d_graph = float((a2.global_master - a.global_master).abs().max())
    d_cross = float((a.global_master - b.global_master).abs().max())
    print(f"LoRA GPT engine: |graph - graph| {d_graph:.3g}, |eager - eager| {d_eager:.3g}, "
          f"|graph - eager| {d_cross:.3g}")
    spread = max(d_eager, d_graph)
    assert d_cross <= max(4 * spread, 1e-6), (d_cross, spread)
    for eng in (a, a2, b, c):
        assert eng.drain_blocks() == [] and eng.host_ledger.verify_chain()
    hits = int(a.val_correct[0])
    ring, size = a.ring_bytes.cpu().numpy(), a.sz["BlockRecord"]
    recs = [parse_block_record(ring, slot * size, 1) for slot in range(8)]
    last = max(recs, key=lambda r: r[0])[2]
    score = float(last["score_rows"][0][0])
    assert a.n_val_targets == 32 * 128
    assert abs(score - hits / a.n_val_targets) <= 1e-6, (score, hits)


def test_engine_refuses_a_net_that_does_not_match_the_lora_config():
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import lm_corpus_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import GPT
    cfg = FLConfig.for_world(1, model="gpt", batch_size=16, samples_per_client=64, learning_rate=1e-3,
                             optimizer="adam", lora_rank=8)
    shard = lm_corpus_like(1, 64, seed=3, seq_len=128, vocab=512, only=0)[0]
    with pytest.raises(ValueError, match="LoRA"):
        GenericFedEngine(cfg, GPT(**GPT_SMALL), shard, rank=0, world=1, device=0)
