"""Poisson-sampled DP-SGD on the GPU (``dpsgd_sampling = "poisson"``): the sampler kernel bit for bit against the
oracle and its overflow counter, padding slots that change nothing, a count-0 step that releases the noise alone,
a sampled MLP step against fp64 per-example autograd of the definition, every DP-SGD family at its capacity, and
engine rounds (graph replay, resume, ledger, accounting).  Needs an H100 (``pytest -m gpu``)."""
import math

import numpy as np
import pytest
import torch

from bflc_demo_b200._native import C
from bflc_demo_b200.ops import dpsgd as D
from bflc_demo_b200.protocol.oracle import DPSGD_SITE, dp_gauss, poisson_sample, poisson_threshold

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
DEV = "cuda"
GPT_SMALL = dict(layers=2, hidden=128, heads=2, ffn=256, vocab=512, max_pos=128)


def _sample_on_device(seed, word, S, thr, cap, steps):
    idx = torch.full((steps, cap), -7, device=DEV, dtype=torch.int32)
    count = torch.full((steps,), -7, device=DEV, dtype=torch.int32)
    over = torch.zeros(1, device=DEV, dtype=torch.int32)
    step = torch.tensor([word], device=DEV, dtype=torch.int32)
    C().dpsgd_poisson_sample(seed, step, S, thr, idx, count, over)
    torch.cuda.synchronize()
    return idx.cpu().numpy(), count.cpu().numpy(), int(over)


@pytest.mark.parametrize("S", [1, 3, 5, 1023, 1024, 1025, 4097, 60000])
@pytest.mark.parametrize("thr", [1, 1 << 28, 1 << 31, (1 << 32) - 1])
def test_sampler_is_bit_exact_against_the_oracle(S, thr):
    seed = 0x0123456789ABCDEF
    for word in (0, 41, -5, 2 ** 31 - 2):
        # cap = S (never overflows), and a small cap that overflows at the larger rates
        for cap in sorted({S, max(1, min(S, 8))}):
            steps = 3
            idx, count, over = _sample_on_device(seed, word, S, thr, cap, steps)
            want_over = 0
            for i in range(steps):
                ri, rc, ro = poisson_sample(seed, (word + i) & 0xFFFFFFFF, S, thr, cap)
                assert count[i] == rc and np.array_equal(idx[i], ri), (S, thr, word, cap, i)
                want_over += int(ro)
            assert over == want_over, (S, thr, word, cap)


def test_sampler_keeps_the_first_cap_and_counts_overflow():
    S, thr, cap = 4096, (1 << 32) - 1, 64        # nearly every record sampled
    idx, count, over = _sample_on_device(5, 0, S, thr, cap, 4)
    assert over == 4 and (count == cap).all()
    for i in range(4):
        full, _, _ = poisson_sample(5, i, S, thr, S)
        assert np.array_equal(idx[i], full[:cap])


# ------------------------------------------------------------------ a step at the capacity
def _mlp_state(seed=5):
    from bflc_demo_b200.models.nets import MLPNet
    net = MLPNet(in_dim=784, hidden=256, n_classes=62)
    P = net.spec.total
    master = torch.zeros(P, device=DEV)
    net.init_(master, seed=seed)
    return net, (master, master.to(BF), torch.zeros(P, device=DEV))


def _mlp_data(n, seed=4):
    from bflc_demo_b200.models.nets import MLPNet
    g = torch.Generator().manual_seed(seed)
    x = MLPNet(784, 256, 62).preprocess(torch.randint(0, 256, (n, 784), generator=g, dtype=torch.uint8).to(DEV))
    return x, torch.randint(0, 62, (n,), generator=g).to(DEV, torch.int32)


def _poisson_grad(net, state, x, y, dp, B, count):
    master, shadow, grad = state
    grad.zero_()
    b = net.bind(master, shadow, grad)
    cap = x.shape[0]
    loss = net.loss(b, x, y)
    dp.begin()
    (loss * (cap / B)).backward()
    dp.finish(grad, 0, n_valid=torch.tensor([count], device=DEV, dtype=torch.int32))
    torch.cuda.synchronize()
    return grad.clone()


def test_padding_slots_change_nothing_and_are_not_dropped():
    net, state = _mlp_state()
    X, Y = _mlp_data(64)
    B, cap, count = 16, 24, 13
    sel = torch.arange(count, device=DEV)
    outs = []
    for pad_src in (0, 40, 63):
        ids = torch.cat([sel, torch.full((cap - count,), pad_src, device=DEV, dtype=torch.long)])
        dp = D.DPSGDStep(net.spec, cap, 0.5, 1.0, 11, torch.zeros(1, device=DEV, dtype=torch.int32), DEV,
                         norm_batch=B)
        outs.append(_poisson_grad(net, state, X[ids], Y[ids], dp, B, count))
        assert int(dp.dropped) == 0 and (dp.c[count:] == 0).all() and (dp.c[:count] > 0).all()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    # a non-finite padding example is masked, not dropped
    Xn = X.clone()
    Xn[40] = float("nan")
    ids = torch.cat([sel, torch.full((cap - count,), 40, device=DEV, dtype=torch.long)])
    dp = D.DPSGDStep(net.spec, cap, 0.5, 1.0, 11, torch.zeros(1, device=DEV, dtype=torch.int32), DEV, norm_batch=B)
    got = _poisson_grad(net, state, Xn[ids], Y[ids], dp, B, count)
    assert int(dp.dropped) == 0 and torch.equal(got, outs[0])


def test_count_zero_step_releases_exactly_the_noise_over_b():
    net, state = _mlp_state()
    X, Y = _mlp_data(24)
    B, clip, z, seed = 16, 0.5, 1.3, 99
    dp = D.DPSGDStep(net.spec, 24, clip, z, seed, torch.zeros(1, device=DEV, dtype=torch.int32), DEV, norm_batch=B)
    got = _poisson_grad(net, state, X, Y, dp, B, 0).cpu().numpy()
    sigma = D.noise_sigma(np.float32(z), np.float32(clip), B)
    want = (np.float32(sigma) * dp_gauss(seed, 0, 0, got.size, DPSGD_SITE)).astype(np.float32)
    assert np.array_equal(got, want)


def test_sampled_mlp_step_against_fp64_per_example_autograd():
    net, state = _mlp_state()
    B, cap, count = 32, 48, 37
    X, Y = _mlp_data(cap, seed=8)
    master, shadow, _ = state
    W = {k: v.double() for k, v in net.spec.views(shadow).items()}
    Pm = net.spec.views(master)
    xs = X.double()

    def per_example(n):
        w1, b1 = W["fc1.w"].clone().requires_grad_(), Pm["fc1.b"].double().clone().requires_grad_()
        w2, b2 = W["fc.w"].clone().requires_grad_(), Pm["fc.b"].double().clone().requires_grad_()
        h = torch.relu(xs[n:n + 1] @ w1.t() + b1)
        loss = torch.nn.functional.cross_entropy(h @ w2.t() + b2, Y[n:n + 1].long())
        return torch.cat([t.reshape(-1) for t in torch.autograd.grad(loss, (w1, b1, w2, b2))])

    g = torch.stack([per_example(n) for n in range(count)])
    norms = g.norm(dim=1)
    clip = float(norms.median())
    ref = (g * (clip / norms).clamp(max=1)[:, None]).sum(0) / B          # 1 / B, never 1 / count or 1 / cap
    dp = D.DPSGDStep(net.spec, cap, clip, 0.0, 0, torch.zeros(1, device=DEV, dtype=torch.int32), DEV, norm_batch=B)
    got = _poisson_grad(net, state, X, Y, dp, B, count)
    V = net.spec.views(got)
    flat = torch.cat([V[k].double().reshape(-1) for k in ("fc1.w", "fc1.b", "fc.w", "fc.b")])
    c = dp.c[:count].double()
    assert (c < 1).any() and (c == 1).any()
    assert float((c - (clip / norms).clamp(max=1)).abs().max()) < 0.03
    assert float((flat - ref).norm() / ref.norm()) < 0.03


def _family(kind):
    from bflc_demo_b200.models.lora import LoRANet
    from bflc_demo_b200.models.nets import GPT, BertBase, LeNet5, ResNet18
    g = torch.Generator().manual_seed(1)
    if kind == "lora_gpt":
        net = LoRANet(GPT(**GPT_SMALL), 8)
        ids = torch.randint(0, 512, (6, 128), generator=g)
        return net, net.preprocess(ids.to(DEV)), torch.randint(0, 512, (6, 128), generator=g).to(DEV, torch.int32), False
    if kind in ("gpt", "bert"):
        net = GPT(**GPT_SMALL) if kind == "gpt" else BertBase(2, layers=2, pad_id=0)
        ids = torch.randint(1, 512, (6, 128), generator=g)
        if kind == "bert":
            ids[:, 96:] = 0
            y = torch.randint(0, 2, (6,), generator=g)
        else:
            y = torch.randint(0, 512, (6, 128), generator=g)
        return net, net.preprocess(ids.to(DEV)), y.to(DEV, torch.int32), False
    net = LeNet5() if kind == "lenet5" else ResNet18(norm="group")
    x = torch.randint(0, 256, (6, 3, 32, 32), generator=g, dtype=torch.uint8)
    return net, net.preprocess(x.to(DEV)), torch.randint(0, 10, (6,), generator=g).to(DEV, torch.int32), True


@pytest.mark.parametrize("kind", ["lora_gpt", "gpt", "bert", "lenet5", "resnet18_gn"])
def test_every_family_padding_is_exact_zeros(kind):
    """At the capacity (6 slots, 4 sampled, B 4), every release path -- linear, Gram, layer norm, embedding,
    convolution and group norm -- leaves the gradient bit-identical whichever record the padding slots read."""
    net, x, y, conv = _family(kind)
    P = net.spec.total
    master = torch.zeros(P, device=DEV)
    net.init_(master, seed=3)
    if hasattr(net, "adapted"):
        V = net.spec.views(master)
        for _, b in net.adapted.values():
            V[b].normal_(0, 0.05, generator=torch.Generator(device=DEV).manual_seed(9))
    state = (master, master.to(BF), torch.zeros(P, device=DEV))
    from bflc_demo_b200.ops import nn as F
    prev = F.set_deterministic(True)
    try:
        outs = []
        for pad in (0, 5):
            ids = torch.tensor([0, 1, 2, 3, pad, pad], device=DEV)
            dp = D.DPSGDStep(net.spec, 6, 1.0, 0.5, 17, torch.zeros(1, device=DEV, dtype=torch.int32), DEV,
                             conv=conv, norm_batch=4)
            grad = state[2]
            grad.zero_()
            b = net.bind(state[0], state[1], grad)
            loss = net.loss(b, x.index_select(0, ids), y.index_select(0, ids))
            dp.begin()
            (loss * 1.5).backward()
            dp.finish(grad, 0, n_valid=torch.tensor([4], device=DEV, dtype=torch.int32))
            torch.cuda.synchronize()
            outs.append(grad.clone())
            assert int(dp.dropped) == 0 and (dp.c[4:] == 0).all()
        assert torch.isfinite(outs[0]).all() and torch.equal(outs[0], outs[1])
    finally:
        F.set_deterministic(prev)


# ------------------------------------------------------------------ engine rounds
def _engine(capture, rounds=0, noise=1.0, seed=7):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import MLPNet
    cfg = FLConfig.for_world(1, model="mlp", batch_size=64, samples_per_client=1024, learning_rate=0.01,
                             optimizer="adam", cuda_graph=capture, dpsgd_clip=1.0, dpsgd_noise=noise,
                             dpsgd_seed=seed, dpsgd_sampling="poisson")
    shard = femnist_like(1, 1024, seed=7, only=0)[0]
    eng = GenericFedEngine(cfg, MLPNet(784, 256, shard.n_classes), shard, rank=0, world=1, device=0)
    if capture:
        eng.capture()
    for _ in range(rounds):
        eng.run_round()
    torch.cuda.synchronize()
    return eng, shard


def test_engine_rounds_replay_equals_eager_and_accounting():
    from bflc_demo_b200.protocol.privacy import binomial_tail, poisson_capacity, poisson_epsilon
    from bflc_demo_b200.utils.checkpoint import plan_counters
    a, _ = _engine(True, rounds=3)
    assert a.capture_error == "" and a.graph_train is not None
    b, _ = _engine(False, rounds=4)          # capture() ran one eager warm-up round
    assert torch.equal(a.global_master, b.global_master)
    assert a.drain_blocks() == [] and b.drain_blocks() == [] and a.host_ledger.verify_chain()
    ps = a.poisson
    q = poisson_threshold(64, 1024) / 2.0 ** 32
    assert ps.q == q and ps.cap == poisson_capacity(1024, q) and ps.eta == binomial_tail(1024, q, ps.cap)
    # the last round's sample is the oracle's
    word = plan_counters(a)[0] - a.steps
    idx, count = ps.idx.cpu().numpy(), ps.count.cpu().numpy()
    for i in range(a.steps):
        ri, rc, _ = poisson_sample(a.dpsgd_seed, word + i, 1024, ps.thr, ps.cap)
        assert count[i] == rc and np.array_equal(idx[i], ri)
    eps, delta = a.privacy_spent_local()
    steps = plan_counters(a)[0]
    want = poisson_epsilon(q, 1.0, steps, a.cfg.dp_delta)
    assert eps == want and delta == a.cfg.dp_delta + (1 + math.exp(eps)) * steps * ps.eta
    assert int(ps.overflow) == 0


def test_checkpoint_resume_reproduces_the_poisson_run(tmp_path):
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import MLPNet
    from bflc_demo_b200.utils.checkpoint import load_checkpoint, save_checkpoint
    eng, shard = _engine(False, rounds=2)
    path = str(tmp_path / "poisson.pt")
    save_checkpoint(path, eng)
    for _ in range(2):
        eng.run_round()
    same = GenericFedEngine(eng.cfg, MLPNet(784, 256, shard.n_classes), shard, rank=0, world=1, device=0)
    load_checkpoint(path, same)
    for _ in range(2):
        same.run_round()
    torch.cuda.synchronize()
    assert torch.equal(same.global_master, eng.global_master)
    assert same.drain_blocks() == [] and same.host_ledger.verify_chain()
    import dataclasses
    other = GenericFedEngine(dataclasses.replace(eng.cfg, dpsgd_sampling="partition"),
                             MLPNet(784, 256, shard.n_classes), shard, rank=0, world=1, device=0)
    with pytest.raises(ValueError, match="sampling"):
        load_checkpoint(path, other)


def test_noiseless_poisson_rounds_sample_with_a_secret_key_and_learn():
    eng, shard = _engine(True, rounds=6, noise=0.0, seed=None)
    assert eng.dpsgd_seed != 0 and eng.poisson.seed == eng.dpsgd_seed
    assert eng.privacy_spent_local()[0] == math.inf
    assert eng.drain_blocks() == []
    assert eng.evaluate(shard) > 2.0 / shard.n_classes


# ------------------------------------------------------------------ every family against fp64 per-example clipping
def _snapshot(monkeypatch):
    fin = D.DPSGDStep.finish

    def spy(self, grad, add, n_valid=None):
        self._snap = list(self._records)
        return fin(self, grad, add, n_valid=n_valid)

    monkeypatch.setattr(D.DPSGDStep, "finish", spy)


# kind -> (records sampled, capacity slots, expected batch size B): cap > B > count or B > cap > count, both n_valid < cap
_SAMPLED = {"lora_gpt": (3, 6, 4), "gpt": (3, 6, 4), "bert_pad": (3, 6, 4), "lenet5": (6, 10, 8), "resnet18": (2, 4, 3)}


def _sampled_setup(kind):
    import test_gpu_dpsgd_conv as TC
    import test_gpu_dpsgd_full as TF
    from bflc_demo_b200.models.lora import LoRANet
    from bflc_demo_b200.models.nets import GPT
    count, cap, B = _SAMPLED[kind]
    n = count + 2
    if kind in ("lenet5", "resnet18"):
        net, _ = TC._net(kind)
        x, y = TC._inputs(net, n, seed=4)
        return net, x, y, True, TC._per_example_fp64, count, cap, B
    if kind == "lora_gpt":
        net = LoRANet(GPT(**GPT_SMALL), 8)
        x, y = TF._inputs("gpt", net, n, seed=4)
    else:
        net, _ = TF._net(kind)
        x, y = TF._inputs(kind, net, n, seed=4)
    return net, x, y, False, TF._per_example_fp64, count, cap, B


def _fresh_state(net):
    P = net.spec.total
    master = torch.zeros(P, device=DEV)
    net.init_(master, seed=3)
    if hasattr(net, "adapted"):        # a non-zero B factor so both adapters get gradients
        V = net.spec.views(master)
        for _, b in net.adapted.values():
            V[b].normal_(0, 0.05, generator=torch.Generator(device=DEV).manual_seed(9))
    return master, master.to(BF), torch.zeros(P, device=DEV)


def _dp_grad(net, state, x, y, dp, scale=1.0, n_valid=None):
    master, shadow, grad = state
    grad.zero_()
    loss = net.loss(net.bind(master, shadow, grad), x, y)
    dp.begin()
    (loss * scale if scale != 1.0 else loss).backward()
    dp.finish(grad, 0, n_valid=n_valid)
    torch.cuda.synchronize()
    return grad.clone()


@pytest.mark.parametrize("kind", ["lora_gpt", "gpt", "bert_pad", "lenet5", "resnet18"])
def test_sampled_step_against_fp64_per_example_clipping(kind, monkeypatch):
    """One Poisson step of every DP-SGD family -- count sampled records in cap slots, the padding reading another
    record, the loss scaled by cap / B, n_valid = count, norm_batch = B -- against the definition on the sampled
    set: (1 / B) sum_n c_n g_n, g_n each sampled example's fp64 gradient.  g_n comes from a plain DP-SGD step
    on the sampled records alone (no padding, no scale, batch = count), its recorded rows materialised in fp64
    as the existing full-model and convolution tests do.  A 1 / cap normalisation, a lost or wrong loss scale or
    a bound at the wrong bsz all fail here: the clip factors must equal the plain step's within 2^-6 and the
    step must be within 2^-6 of the fp64 sum over B."""
    from bflc_demo_b200.ops import nn as F
    _snapshot(monkeypatch)
    net, x, y, conv, per_example, count, cap, B = _sampled_setup(kind)
    state = _fresh_state(net)
    word = torch.zeros(1, device=DEV, dtype=torch.int32)
    prev = F.set_deterministic(True)
    try:
        xs, ys = x[:count], y[:count]
        probe = D.DPSGDStep(net.spec, count, 1e30, 0.0, 0, word, DEV, conv=conv)
        _dp_grad(net, state, xs, ys, probe)
        g = per_example(probe, net, state, count)
        norms = g.norm(dim=1)
        clip = float(norms.median())
        plain = D.DPSGDStep(net.spec, count, clip, 0.0, 0, word, DEV, conv=conv)
        _dp_grad(net, state, xs, ys, plain)
        ids = torch.tensor(list(range(count)) + [count + 1] * (cap - count), device=DEV)
        dp = D.DPSGDStep(net.spec, cap, clip, 0.0, 0, word, DEV, conv=conv, norm_batch=B)
        got = _dp_grad(net, state, x.index_select(0, ids), y.index_select(0, ids), dp, cap / B,
                       torch.tensor([count], device=DEV, dtype=torch.int32)).double()
    finally:
        F.set_deterministic(prev)
    c, c_plain = dp.c[:count].double(), plain.c.double()
    assert (dp.c[count:] == 0).all() and int(dp.dropped) == 0
    assert (c_plain < 1).any(), c_plain
    ratio = c / c_plain
    print(kind, "c / c_plain", ratio.tolist())
    assert float((ratio - 1).abs().max()) < 2 ** -6
    ref = (g * c[:, None]).sum(0) / B
    rel = float((got - ref).norm() / ref.norm())
    print(kind, "relative error of the sampled step", rel)
    assert rel < 2 ** -6


# ------------------------------------------------------------------ engine rounds of the other families
def _family_engine(kind, capture, rounds):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import cifar_like, lm_corpus_like, tokens_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.lora import lora_net_from_config
    from bflc_demo_b200.models.nets import GPT, BertBase, LeNet5
    common = dict(cuda_graph=capture, dpsgd_clip=1.0, dpsgd_noise=1.0, dpsgd_seed=3, dpsgd_sampling="poisson")
    if kind == "lora_gpt":
        cfg = FLConfig.for_world(1, model="gpt", batch_size=8, samples_per_client=32, learning_rate=2e-3,
                                 optimizer="adam", lora_rank=8, **common)
        shard = lm_corpus_like(1, 32, seed=2, seq_len=128, vocab=512, only=0)[0]
        net = lora_net_from_config(cfg, GPT(**GPT_SMALL))
    elif kind == "bert_pad":
        cfg = FLConfig.for_world(1, model="bert", batch_size=4, samples_per_client=16, learning_rate=2e-3,
                                 dpsgd_full_model=True, **common)
        shard = tokens_like(1, 16, seed=2, seq_len=128, min_len=32)[0]
        net = BertBase(shard.n_classes, layers=2, pad_id=0)
    else:
        cfg = FLConfig.for_world(1, model="lenet5", batch_size=16, samples_per_client=64, learning_rate=0.02,
                                 dpsgd_conv=True, **common)
        shard = cifar_like(1, 64, seed=2)[0]
        net = LeNet5()
    eng = GenericFedEngine(cfg, net, shard, rank=0, world=1, device=0)
    if capture:
        eng.capture()
    for _ in range(rounds):
        eng.run_round()
    torch.cuda.synchronize()
    return eng


@pytest.mark.parametrize("kind", ["lora_gpt", "bert_pad", "lenet5"])
def test_engine_rounds_of_every_gather_path(kind):
    """The engine's Poisson steps on token ids (GPT's per-position targets and row losses, BERT's key lengths
    re-derived from the gathered ids) and NHWC images: captured rounds equal eager ones bit for bit, the ledgers
    agree, and the published avg_cost is a finite mean loss."""
    from bflc_demo_b200.engine.base import parse_block_record
    a = _family_engine(kind, True, 2)
    assert a.capture_error == "" and a.graph_train is not None
    b = _family_engine(kind, False, 3)
    assert torch.equal(a.global_master, b.global_master)
    assert a.drain_blocks() == [] and b.drain_blocks() == [] and a.host_ledger.verify_chain()
    ring = a.ring_bytes.cpu().numpy()
    epoch = a.read_state()["epoch"]
    from bflc_demo_b200.engine.base import BLOCK_RECORD
    _, _, rnd = parse_block_record(ring, ((epoch - 1) % (len(ring) // BLOCK_RECORD.size)) * BLOCK_RECORD.size, 1)
    cost = rnd["avg_cost"][0]
    assert math.isfinite(cost) and cost > 0, rnd["avg_cost"]
    assert rnd["n_samples"][0] == a.S          # the nominal count, as without sampling
    assert int(a.poisson.overflow) == 0 and torch.isfinite(a.global_master).all()


def test_sampler_compare_at_a_records_own_uniform():
    """thr = u_j leaves record j out and thr = u_j + 1 takes it, on the device as in the oracle."""
    from bflc_demo_b200.protocol.oracle import DPSGD_SAMPLE_SITE, philox4x32_10
    S, seed, word = 1000, 0xABCDEF, 12
    g = np.arange(S // 4, dtype=np.uint32)
    w = philox4x32_10((g, np.zeros_like(g), np.full(g.shape, word, np.uint32),
                       np.full(g.shape, DPSGD_SAMPLE_SITE, np.uint32)), seed & 0xFFFFFFFF, seed >> 32)
    u = np.stack(w, axis=1).reshape(-1)
    for j in (0, 5, 498, 999):
        for thr in (int(u[j]), int(u[j]) + 1):
            if not 0 < thr < 1 << 32:
                continue
            idx, count, _ = _sample_on_device(seed, word, S, thr, S, 1)
            ri, rc, _ = poisson_sample(seed, word, S, thr, S)
            assert count[0] == rc and np.array_equal(idx[0], ri)
            assert (j in idx[0][:count[0]]) == (thr > u[j])
