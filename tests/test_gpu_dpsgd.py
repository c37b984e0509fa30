"""DP-SGD local training on the GPU (ops/dpsgd.py, csrc/kernels/dpsgd_kernels.cu): the per-example norm
kernels against fp64, the clip factors against their fp32 host mirror, a step with C above every bound
against the same step without DP-SGD, the clipped gradient against fp64 per-example autograd, the
certified bound at B = 1, the noise against the host sampler, and engine rounds (graph replay, resume,
ledger).  Needs an H100 (``pytest -m gpu``)."""
import math

import numpy as np
import pytest
import torch

from bflc_demo_b200._native import C
from bflc_demo_b200.ops import dpsgd as D
from bflc_demo_b200.ops import nn as F
from bflc_demo_b200.protocol.oracle import DPSGD_SITE, dp_gauss

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
DEV = "cuda"
GPT_SMALL = dict(layers=2, hidden=128, heads=2, ffn=256, vocab=512, max_pos=128)


def _pe_sq64(A, Bm, R):
    """fp64 ||A_n^T Bm_n||^2 per 64-row tile of A's columns: [tiles, n_ex]."""
    a, b = A.double(), Bm.double()
    n_ex, tiles = A.shape[0] // R, (A.shape[1] + 63) // 64
    out = torch.empty(tiles, n_ex, dtype=torch.float64, device=A.device)
    for n in range(n_ex):
        p = a[n * R:(n + 1) * R].t() @ b[n * R:(n + 1) * R]
        for t in range(tiles):
            out[t, n] = (p[64 * t:64 * t + 64] ** 2).sum()
    return out


def _canaried(n):
    buf = torch.full((n + 64,), float("nan"), device=DEV)
    return buf, buf[32:32 + n]


@pytest.mark.parametrize("r", [8, 16, 64])
@pytest.mark.parametrize("R, n_ex, wide", [(64, 3, 768), (128, 16, 62), (512, 1, 3072), (128, 3, 200),
                                           (64, 16, 3072)])
def test_pe_norm_against_fp64_with_canaries_and_reruns(r, R, n_ex, wide):
    g = torch.Generator(device=DEV).manual_seed(r * 1000 + R + wide)
    A = torch.randn(n_ex * R, wide, device=DEV, generator=g).to(BF)
    Bm = torch.randn(n_ex * R, r, device=DEV, generator=g).to(BF)
    tiles = (wide + 63) // 64
    buf, out = _canaried(tiles * n_ex)
    C().dpsgd_pe_norm(A, Bm, R, out)
    torch.cuda.synchronize()
    ref = _pe_sq64(A, Bm, R).reshape(-1)
    assert torch.isnan(buf[:32]).all() and torch.isnan(buf[32 + tiles * n_ex:]).all()
    assert float(((out.double() - ref).abs() / ref.clamp_min(1e-30)).max()) < 1e-5
    again = torch.full_like(out, float("nan"))
    C().dpsgd_pe_norm(A, Bm, R, again)
    assert torch.equal(out, again)


def test_pe_norm_is_exact_on_integers_and_reads_strided_views():
    g = torch.Generator(device=DEV).manual_seed(5)
    R, n_ex, wide, r = 64, 3, 200, 8
    base = torch.randint(-1, 2, (n_ex * R, 256), device=DEV, generator=g).to(BF)
    A = base[:, 3:3 + wide]                       # pitch 256, an unaligned start: the scalar path
    Bm = torch.randint(-1, 2, (n_ex * R, r), device=DEV, generator=g).to(BF)
    out = torch.empty((wide + 63) // 64 * n_ex, device=DEV)
    C().dpsgd_pe_norm(A, Bm, R, out)
    assert torch.equal(out.double(), _pe_sq64(A, Bm, R).reshape(-1))


@pytest.mark.parametrize("R", [1, 64, 128])
def test_pe_rows_against_fp64(R):
    g = torch.Generator(device=DEV).manual_seed(R)
    n_ex = 16
    A = torch.randint(-3, 4, (n_ex * R, 200), device=DEV, generator=g).to(BF)
    Bm = torch.randint(-3, 4, (n_ex * R, 62), device=DEV, generator=g).to(BF)
    if R == 1:
        Bm[0] = 0         # example 0's operand row is zero: its norm is the bias term alone
    ab = torch.empty(n_ex, device=DEV)
    sq = torch.empty(n_ex, device=DEV) if R == 1 else None
    bias = 1.0 if R == 1 else 0.0
    C().dpsgd_pe_rows(A, Bm, R, bias, sq, ab)
    ra = (A.double() ** 2).sum(1)
    rb = (Bm.double() ** 2).sum(1) + bias
    ref_ab = (ra.sqrt() * rb.sqrt()).view(n_ex, R).sum(1)
    assert float(((ab.double() - ref_ab).abs() / ref_ab).max()) < 1e-6
    if R == 1:   # ||dz x^T||^2 + ||dz||^2 of integer rows: exact
        assert torch.equal(sq.double(), ra * rb)
        assert float(sq[0]) == float(ra[0]) > 0      # without the bias term it would be 0


def test_clip_factors_match_the_host_mirror_bit_for_bit():
    rng = np.random.default_rng(0)
    n_sq, n_ab, B = 7, 3, 300
    sq = (rng.random((n_sq, B)) * 10 ** rng.uniform(-6, 4, (n_sq, B))).astype(np.float32)
    ab = (rng.random((n_ab, B)) * 10 ** rng.uniform(-4, 2, (n_ab, B))).astype(np.float32)
    sq[0, 5], ab[1, 6], sq[2, 7], sq[3, 7] = np.inf, np.nan, np.float32(3e38), np.float32(3e38)
    for clip in (1e30, 0.5, 3.0):
        c = torch.empty(B, device=DEV)
        dropped = torch.zeros(1, device=DEV, dtype=torch.int32)
        C().dpsgd_clip(torch.from_numpy(sq).to(DEV), n_sq, torch.from_numpy(ab).to(DEV), n_ab, B, float(B),
                       clip, c, dropped)
        want = D.clip_factors(sq, ab, B, clip)
        assert np.array_equal(c.cpu().numpy().view(np.uint32), want.view(np.uint32))
        assert int(dropped) == int((want == 0).sum()) == 3      # c = 0 exactly when the bound is not finite
        assert want[5] == 0 and want[6] == 0 and want[7] == 0
        if clip == 1e30:
            assert (want[np.isfinite(sq.sum(0)) & np.isfinite(ab.sum(0)) & (sq.max(0) < 1e30)] == 1).all()


def test_scale_rows_and_fixed_order_colsum():
    g = torch.Generator(device=DEV).manual_seed(1)
    X = torch.randn(48, 70, device=DEV, generator=g).to(BF)
    c = torch.tensor([1.0, 0.3, 0.0], device=DEV)
    out = torch.empty_like(X)
    C().dpsgd_scale_rows(X, c, 16, out)
    want = (X.float() * c.repeat_interleave(16)[:, None]).to(BF)
    assert torch.equal(out, want)
    gb1, gb2 = torch.ones(70, device=DEV), torch.ones(70, device=DEV)
    C().dpsgd_colsum(out, gb1)
    C().dpsgd_colsum(out, gb2)
    assert torch.equal(gb1, gb2)
    ref = 1 + out.double().sum(0)
    assert float((gb1.double() - ref).abs().max()) <= 48 * 2 ** -23 * float(out.double().abs().sum(0).max() + 1)


def test_noise_equals_the_host_sampler_and_is_fresh_per_step():
    P, seed, sigma = 1003, 0x1234567890ABCDEF, 0.125
    step = torch.tensor([41], device=DEV, dtype=torch.int32)
    outs = []
    for add in (0, 1):
        g = torch.zeros(P, device=DEV)
        C().dpsgd_noise(g, seed, step, add, sigma)
        want = np.float32(sigma) * dp_gauss(seed, 41 + add, 0, P, DPSGD_SITE)
        assert np.array_equal(g.cpu().numpy(), want.astype(np.float32))
        outs.append(g)
    assert not torch.equal(outs[0], outs[1])
    assert not np.array_equal(dp_gauss(seed, 41, 0, P, DPSGD_SITE), dp_gauss(seed, 41, 0, P))


# ------------------------------------------------------------------ model steps
def _net(kind):
    from bflc_demo_b200.models.lora import LoRANet
    from bflc_demo_b200.models.nets import GPT, BertBase, MLPNet
    if kind == "mlp":
        return MLPNet(in_dim=784, hidden=256, n_classes=62), 64
    if kind == "gpt":
        return LoRANet(GPT(**GPT_SMALL), 8), 4
    return LoRANet(BertBase(2, layers=2, pad_id=0 if kind == "bert_pad" else None), 8), 4


def _inputs(kind, net, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    if kind == "mlp":
        x = net.preprocess(torch.randint(0, 256, (B, 784), generator=g, dtype=torch.uint8).to(DEV))
        return x, torch.randint(0, 62, (B,), generator=g).to(DEV, torch.int32)
    if kind == "gpt":
        ids = torch.randint(0, 512, (B, 128), generator=g)
        return net.preprocess(ids.to(DEV)), torch.randint(0, 512, (B, 128), generator=g).to(DEV, torch.int32)
    ids = torch.randint(1, 1000, (B, 128), generator=g)
    if kind == "bert_pad":
        for n in range(B):
            ids[n, 32 + 16 * n:] = 0
    return net.preprocess(ids.to(DEV)), torch.randint(0, 2, (B,), generator=g).to(DEV, torch.int32)


def _state(net, seed=3):
    P = net.spec.total
    master = torch.zeros(P, device=DEV)
    net.init_(master, seed=seed)
    if hasattr(net, "adapted"):        # a non-zero B factor so both adapters get gradients
        V = net.spec.views(master)
        for _, b in net.adapted.values():
            V[b].normal_(0, 0.05, generator=torch.Generator(device=DEV).manual_seed(9))
    return master, master.to(BF), torch.zeros(P, device=DEV)


def _grad(net, x, y, state, dp=None):
    master, shadow, grad = state
    grad.zero_()
    b = net.bind(master, shadow, grad)
    loss = net.loss(b, x, y)
    if dp is None:
        loss.backward()
    else:
        dp.begin()
        loss.backward()
        dp.finish(grad, 0)
    torch.cuda.synchronize()
    return grad.clone()


def _step_word():
    return torch.zeros(1, device=DEV, dtype=torch.int32)


@pytest.mark.parametrize("kind", ["mlp", "bert", "bert_pad", "gpt"])
def test_unclipped_noiseless_step_is_the_plain_step(kind, monkeypatch):
    """C above every bound and z = 0: c = 1, so every weight and adapter gradient is bit-identical to the
    step without DP-SGD run through the same single-writer GEMM (without DP-SGD, ops.nn splits small
    weight-gradient GEMMs over K with fp32 atomics, whose order is not fixed), and a rerun of the DP-SGD
    step gives the same bits.  A bias gradient is the sum of the bf16 rows the weight GEMM reads, where
    the path without DP-SGD sums the fp32 values before rounding: they agree within 2^-8 sum_r |dz_r|."""
    net, B = _net(kind)
    x, y = _inputs(kind, net, B)
    state = _state(net)
    dp = D.DPSGDStep(net.spec, B, 1e30, 0.0, 0, _step_word(), DEV)
    col_abs = {}
    record = D.DPSGDStep.record

    def spy(self, dz, op, gw, gb):
        if gb is not None:
            col_abs[gb.data_ptr()] = dz.double().abs().sum(0)
        return record(self, dz, op, gw, gb)

    monkeypatch.setattr(D.DPSGDStep, "record", spy)
    got = _grad(net, x, y, state, dp)
    assert torch.equal(got, _grad(net, x, y, state, dp))
    assert torch.equal(dp.c, torch.ones(B, device=DEV)) and int(dp.dropped) == 0
    monkeypatch.setattr(F, "_split_k", lambda *a: 1)
    plain = _grad(net, x, y, state)
    G_, P_ = net.spec.views(got), net.spec.views(plain)
    for e in net.spec.entries:
        if len(e.shape) == 2:
            assert torch.equal(G_[e.name], P_[e.name]), e.name
        else:
            bound = 2 ** -8 * col_abs[net.spec.views(state[2])[e.name].data_ptr()] + 1e-7
            assert ((G_[e.name].double() - P_[e.name].double()).abs() <= bound).all(), e.name
    assert float(got.abs().sum()) > 0


def test_clipped_mlp_gradient_against_fp64_per_example_autograd():
    from bflc_demo_b200.models.nets import MLPNet
    net, B = MLPNet(in_dim=784, hidden=256, n_classes=62), 32
    x, y = _inputs("mlp", net, B, seed=4)
    state = _state(net, seed=5)
    master, shadow, _ = state
    W = {k: v.double() for k, v in net.spec.views(shadow).items()}
    Pm = net.spec.views(master)
    xs = x.double()

    def per_example(n):
        w1, b1 = W["fc1.w"].clone().requires_grad_(), Pm["fc1.b"].double().clone().requires_grad_()
        w2, b2 = W["fc.w"].clone().requires_grad_(), Pm["fc.b"].double().clone().requires_grad_()
        h = torch.relu(xs[n:n + 1] @ w1.t() + b1)
        loss = torch.nn.functional.cross_entropy(h @ w2.t() + b2, y[n:n + 1].long())
        return torch.cat([t.reshape(-1) for t in torch.autograd.grad(loss, (w1, b1, w2, b2))])

    g = torch.stack([per_example(n) for n in range(B)])
    norms = g.norm(dim=1)
    clip = float(norms.median())
    ref = (g * (clip / norms).clamp(max=1)[:, None]).sum(0) / B
    dp = D.DPSGDStep(net.spec, B, clip, 0.0, 0, _step_word(), DEV)
    got = _grad(net, x, y, state, dp)
    V = net.spec.views(got)
    flat = torch.cat([V[k].double().reshape(-1) for k in ("fc1.w", "fc1.b", "fc.w", "fc.b")])
    c = dp.c.double()
    assert (c < 1).any() and (c == 1).any()
    assert float((c - (clip / norms).clamp(max=1)).abs().max()) < 0.03
    assert float((flat - ref).norm() / ref.norm()) < 0.03


@pytest.mark.parametrize("kind", ["mlp", "gpt"])
def test_single_example_contribution_is_within_the_clip(kind):
    net, _ = _net(kind)
    x, y = _inputs(kind, net, 1, seed=6)
    state = _state(net)
    unclipped = _grad(net, x, y, state, D.DPSGDStep(net.spec, 1, 1e30, 0.0, 0, _step_word(), DEV))
    clip = 0.25 * float(unclipped.double().norm())
    got = _grad(net, x, y, state, D.DPSGDStep(net.spec, 1, clip, 0.0, 0, _step_word(), DEV))
    n = float(got.double().norm())
    print(f"{kind}: B = 1 contribution {n / clip:.4f} C")
    # the certified bound's rounding slack keeps the clipped contribution a little under C (more for many
    # tokens, where sum_t ||dz_t|| ||x_t|| exceeds the gradient's norm)
    assert 0.5 * clip < n <= clip, (n, clip)


# ------------------------------------------------------------------ engine rounds
def _engine(capture, rounds=0, noise=0.5, **kw):
    """A 1-GPU generic MLP engine with DP-SGD (C 1, Adam; B 256: noise std z / 256 per coordinate)."""
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import MLPNet
    cfg = FLConfig.for_world(1, model="mlp", batch_size=256, samples_per_client=1024, learning_rate=0.01,
                             optimizer="adam", cuda_graph=capture, dpsgd_clip=1.0, dpsgd_noise=noise, dpsgd_seed=7,
                             **kw)
    shard = femnist_like(1, 1024, seed=7, only=0)[0]
    eng = GenericFedEngine(cfg, MLPNet(784, 256, shard.n_classes), shard, rank=0, world=1, device=0)
    if capture:
        eng.capture()
    for _ in range(rounds):
        eng.run_round()
    torch.cuda.synchronize()
    return eng, shard


def test_replayed_rounds_equal_eager_rounds_bit_for_bit():
    a, _ = _engine(True, rounds=3)
    assert a.capture_error == "" and a.graph_train is not None
    b, _ = _engine(False, rounds=4)          # capture() ran one eager warm-up round
    assert torch.equal(a.global_master, b.global_master)
    assert a.drain_blocks() == [] and b.drain_blocks() == [] and a.host_ledger.verify_chain()
    eps0, delta = a.privacy_spent_local()
    assert delta == a.cfg.dp_delta and math.isfinite(eps0) and eps0 > 0
    a.run_round()
    assert a.privacy_spent_local()[0] > eps0


def test_checkpoint_resume_reproduces_the_run_and_refuses_another_key(tmp_path):
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import MLPNet
    from bflc_demo_b200.utils.checkpoint import load_checkpoint, save_checkpoint
    eng, shard = _engine(False, rounds=2)
    path = str(tmp_path / "dpsgd.pt")
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
    other_cfg = dataclasses.replace(eng.cfg, dpsgd_seed=8)
    other = GenericFedEngine(other_cfg, MLPNet(784, 256, shard.n_classes), shard, rank=0, world=1, device=0)
    with pytest.raises(ValueError, match="DP-SGD noise key"):
        load_checkpoint(path, other)


def test_noisy_mlp_still_learns_above_chance():
    eng, _ = _engine(True, rounds=8, noise=0.5)
    from bflc_demo_b200.data.synthetic import femnist_like
    held_out = femnist_like(2, 1024, seed=7, only=1)[0]   # the same classes, another client's samples
    acc = eng.evaluate(held_out)
    print(f"DP-SGD MLP (C 1, z 0.5) held-out accuracy after 9 rounds: {acc:.3f}")
    assert acc > 0.5          # chance is 1/62
    assert eng.drain_blocks() == []


@pytest.mark.parametrize("kind", ["gpt"])
def test_lora_gpt_rounds_are_bit_reproducible(kind):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import lm_corpus_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.lora import LoRANet
    from bflc_demo_b200.models.nets import GPT
    shard = lm_corpus_like(1, 32, seed=3, seq_len=128, vocab=512, only=0)[0]

    def run(capture):
        cfg = FLConfig.for_world(1, model="gpt", batch_size=8, samples_per_client=32, learning_rate=3e-3,
                                 cuda_graph=capture, lora_rank=8, dpsgd_clip=0.5, dpsgd_noise=1.0, dpsgd_seed=3)
        eng = GenericFedEngine(cfg, LoRANet(GPT(**GPT_SMALL), 8), shard, rank=0, world=1, device=0)
        if capture:
            eng.capture()
        for _ in range(3 if capture else 4):
            eng.run_round()
        torch.cuda.synchronize()
        assert eng.drain_blocks() == [] and eng.host_ledger.verify_chain()
        return eng.global_master.clone()

    assert torch.equal(run(True), run(False))


def test_non_finite_example_is_dropped_and_the_step_stays_finite():
    """One MLP example with a NaN feature: its bound is not finite, so c = 0, ``dropped`` counts it, and
    its output-gradient and operand rows enter the weight GEMMs and bias sums as exact zeros.  The step's
    gradient is then that of the other examples (scaled by 1 / B, B counting the dropped one), up to the
    bf16 rounding of dlogits, whose 1 / M scale differs between the two batches."""
    net, B = _net("mlp")
    x, y = _inputs("mlp", net, B, seed=8)
    state = _state(net)
    bad = x.clone()
    bad[5, 100] = float("nan")
    dp = D.DPSGDStep(net.spec, B, 1e30, 0.0, 0, _step_word(), DEV)
    got = _grad(net, bad, y, state, dp)
    assert int(dp.dropped) == 1 and float(dp.c[5]) == 0.0 and torch.isfinite(got).all()
    keep = torch.arange(B, device=DEV) != 5
    rest = _grad(net, x[keep], y[keep], state, D.DPSGDStep(net.spec, B - 1, 1e30, 0.0, 0, _step_word(), DEV))
    want = rest.double() * (B - 1) / B
    assert float((got.double() - want).norm() / want.norm()) < 2 ** -8
    assert float(got.abs().sum()) > 0


def test_noise_is_scaled_per_example_not_per_row():
    """LoRA GPT, B 4 examples of 128 tokens: the noise a step adds is (z C / B) xi on every coordinate, keyed
    by the step word plus the step index, not z C / (B S)."""
    net, B = _net("gpt")
    x, y = _inputs("gpt", net, B, seed=9)
    state = _state(net)
    clip, z, seed, add = 0.5, 2.0, 0xC0FFEE, 3
    word = torch.tensor([40], device=DEV, dtype=torch.int32)
    clean = D.DPSGDStep(net.spec, B, clip, 0.0, seed, word, DEV)
    noisy = D.DPSGDStep(net.spec, B, clip, z, seed, word, DEV)

    def step(dp):
        master, shadow, grad = state
        grad.zero_()
        loss = net.loss(net.bind(master, shadow, grad), x, y)
        dp.begin()
        loss.backward()
        dp.finish(grad, add)
        torch.cuda.synchronize()
        return grad.clone()

    diff = (step(noisy).double() - step(clean).double()).cpu()
    xi = torch.from_numpy(dp_gauss(seed, 40 + add, 0, net.spec.total, DPSGD_SITE)).double()
    want = z * clip / B * xi
    assert float((diff - want).abs().max()) < 1e-6 * float(want.abs().max())


def test_lora_gpt_rounds_above_every_bound_equal_rounds_without_dpsgd(monkeypatch):
    """LoRA GPT has no trainable bias, so with C above every bound and z = 0 its uploads are bit-identical
    to rounds without DP-SGD over whole rounds (the latter's weight-gradient GEMMs run single-writer, as
    DP-SGD's do: their default split-K adds partial sums with fp32 atomics in no fixed order)."""
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import lm_corpus_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.lora import LoRANet
    from bflc_demo_b200.models.nets import GPT
    monkeypatch.setattr(F, "_split_k", lambda *a: 1)
    shard = lm_corpus_like(1, 32, seed=3, seq_len=128, vocab=512, only=0)[0]

    def run(**kw):
        cfg = FLConfig.for_world(1, model="gpt", batch_size=8, samples_per_client=32, learning_rate=3e-3,
                                 lora_rank=8, **kw)
        eng = GenericFedEngine(cfg, LoRANet(GPT(**GPT_SMALL), 8), shard, rank=0, world=1, device=0)
        eng.capture()
        for _ in range(3):
            eng.run_round()
        torch.cuda.synchronize()
        assert eng.capture_error == "" and eng.drain_blocks() == []
        if eng.dpsgd is not None:
            assert torch.equal(eng.dpsgd.c, torch.ones_like(eng.dpsgd.c))
        return eng.global_master.clone(), eng.work_master.clone()

    on, off = run(dpsgd_clip=1e30), run()
    assert torch.equal(on[0], off[0]) and torch.equal(on[1], off[1])
    assert float(on[0].abs().sum()) > 0
