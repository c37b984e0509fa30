"""The GPT decoder (``models.nets.GPT``) on the hand-written kernels against an independent float64
GPT, and the generic engine training it.  The method and the checkers are those of
``test_gpu_model_conformance.py``, whose recorder and per-op stage checks run here on GPT.

* Stages: one training forward + backward under that suite's ``Recorder``; every recorded op is
  checked from its own recorded operands -- linear (output, dx, weight and bias gradients), layer
  norm, residual add and hidden dropout by that suite's ``stage_*`` checks; the causal attention core
  against ``test_gpu_attention_causal``'s fp64 reference and bounds (O, dQ, dK, dV); the embedding
  output and position gradient; the LM head's loss, dh, and the tied ``emb.word`` gradient, which must
  equal the embedding scatter plus the head's ``dlogits^T h``.
* End to end: the loss and every gradient view of the flat buffer after one backward from zero,
  against an independent fp64 GPT written here (``fp64_gpt``), ``||kernel - fp64|| <= 2
  ||emulation - fp64|| + floor`` per view, the emulation rounding to bf16 at every point the kernels
  store bf16 (activations, their gradients, P and dS in attention, dlogits).  Views that are zero in
  exact arithmetic (the key biases) are reported, not held to the ratio.
* Causality through the whole model: perturbing token t leaves every output row at positions < t
  bit-identical and changes position t.
* Dropout: the model draws at the site ids it documents (``8 layer + kind``), every site draws a
  different mask, the same (seed, step) reproduces the loss bit for bit and a new step changes it;
  ``correct`` never drops.
* ``correct`` equals the fp64 argmax count exactly, on targets set to the fp64 argmax for half of
  the rows whose top-2 margin exceeds the logits' error bound and to the least likely token for
  every other row.
* 1-GPU GenericFedEngine rounds: no ledger mismatch, ``verify_chain``, committee scores = hits /
  (n_val * S), test next-token accuracy well above chance.  Graph capture: with lr = 0 one replay
  of the captured training pass gives the eager pass's loss bit for bit, and the captured validation
  the eager hit count.  Whole trained rounds are compared against eager only to within the spread
  of two eager runs: the embedding backward accumulates its fp32 table gradient with atomics, so two
  runs may add in a different order.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as TF
from torch.autograd import Function

import test_gpu_model_conformance as MC
from test_gpu_attention_causal import bwd_bounds as causal_bwd_bounds
from test_gpu_attention_causal import causal_mask
from test_gpu_attention_causal import fwd_bounds as causal_fwd_bounds
from test_gpu_attention_causal import ref_bwd as causal_ref_bwd
from test_gpu_attention_causal import ref_fwd as causal_ref_fwd
from test_gpu_attention_conformance import violations as attn_violations
from test_gpu_lm_head import xent_bounds

gpu = pytest.mark.gpu
pytestmark = gpu
F64, BF16 = torch.float64, torch.bfloat16
U, ULP, BF_U = 2.0 ** -24, 2.0 ** -23, 2.0 ** -8
RATIO = 2.0
SMALL = dict(layers=2, hidden=128, heads=2, ffn=256, vocab=512, max_pos=128)


def make(dropout=0.0, seed=1):
    """A small GPT with non-trivial biases and norm parameters, on flat buffers."""
    from bflc_demo_b200.models.nets import GPT
    net = GPT(dropout=dropout, **SMALL)
    master = torch.empty(net.spec.total)
    net.init_(master, seed=seed)
    g = torch.Generator().manual_seed(seed + 9)
    for k, v in net.spec.views(master).items():
        if k.endswith(".b") or k.endswith(".beta"):
            v.copy_(torch.randn(v.shape, generator=g) * 0.02)
        elif k.endswith(".gamma"):
            v.copy_(1 + torch.randn(v.shape, generator=g) * 0.05)
    master = master.cuda()
    shadow = master.to(BF16)
    grad = torch.zeros_like(master)
    return net, net.bind(master, shadow, grad), master, shadow, grad


def data(B=4, S=128, seed=0):
    from bflc_demo_b200.data.synthetic import lm_corpus_like
    sh = lm_corpus_like(1, B, seed=seed, seq_len=S, vocab=SMALL["vocab"])[0]
    return sh.x.cuda().to(torch.int32), sh.y.cuda().to(torch.int32)


# ------------------------------------------------------------------ independent fp64 GPT
class CausalAttnEmu(Function):
    """The fused causal kernels' storage points on q, k, v [B, H, S, 64] fp64: P rounded to bf16
    before P V, O stored in bf16; the backward takes delta from the stored O and rounds dS."""

    @staticmethod
    def forward(ctx, q, k, v, scale):
        S = q.shape[2]
        mask = torch.ones(S, S, dtype=torch.bool, device=q.device).tril()
        P = torch.softmax((q @ k.transpose(-1, -2) * scale).masked_fill(~mask, -math.inf), -1)
        O = MC._bf(MC._bf(P) @ v)
        ctx.save_for_backward(q, k, v, P, O)
        ctx.scale = scale
        return O

    @staticmethod
    def backward(ctx, dO):
        q, k, v, P, O = ctx.saved_tensors
        dv = MC._bf(P).transpose(-1, -2) @ dO
        dP = dO @ v.transpose(-1, -2)
        dS = MC._bf(P * (dP - (dO * O).sum(-1, keepdim=True)) * ctx.scale)
        return dS @ k, dS.transpose(-1, -2) @ q, dv, None


def fp64_gpt(net, Pd, ids, y, m):
    """Pre-LN GPT-2 written from its documented architecture on fp64 leaves ``Pd`` (shadow values for
    GEMM weights and embeddings, master values for the rest); ``m`` a ``Model64`` (rounding hooks).
    The head is tied: ``emb.word`` is one leaf used twice."""
    B, S = ids.shape
    Hd, H = net.Hd, net.heads
    ids = ids.long()

    def ln(t, name):
        return m.r(TF.layer_norm(t, (Hd,), Pd[f"{name}.gamma"], Pd[f"{name}.beta"], 1e-12))

    def heads(t):
        return t.view(B, S, H, 64).transpose(1, 2)

    x = m.r(Pd["emb.word"][ids.reshape(-1)] + Pd["emb.pos"][torch.arange(S, device=ids.device).repeat(B)])
    for i in range(net.L):
        e = f"dec{i}"
        a = ln(x, f"{e}.ln1")
        q, k, v = (heads(m.linear(a, Pd[f"{e}.{n}.w"], Pd[f"{e}.{n}.b"])) for n in "qkv")
        if m.emul:
            att = CausalAttnEmu.apply(q, k, v, 0.125)
        else:
            att = TF.scaled_dot_product_attention(q, k, v, is_causal=True, scale=0.125)
        att = m.r(att.transpose(1, 2).reshape(B * S, Hd))
        x = m.r(x + m.linear(att, Pd[f"{e}.o.w"], Pd[f"{e}.o.b"]))
        f = m.linear(ln(x, f"{e}.ln2"), Pd[f"{e}.ff1.w"], Pd[f"{e}.ff1.b"], MC.G.ACT_GELU)
        x = m.r(x + m.linear(f, Pd[f"{e}.ff2.w"], Pd[f"{e}.ff2.b"]))
    h = ln(x, "ln_f")
    z = m.rg(h @ Pd["emb.word"].t())                 # fp32 logits; dlogits stored in bf16
    return TF.cross_entropy(z, y.reshape(-1).long())


def fp64_run(net, master, shadow, ids, y, emul):
    Pd = MC.fp64_params(net, master, shadow, "cuda")
    loss = fp64_gpt(net, Pd, ids, y, MC.Model64(emul))
    loss.backward()
    return loss.detach(), {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in Pd.items()}


def test_gpt_loss_and_every_gradient_end_to_end_against_fp64():
    net, b, master, shadow, flat = make()
    ids, y = data()
    m0 = master.clone()
    loss = net.loss(b, ids, y)
    loss.backward()
    torch.cuda.synchronize()
    f64 = fp64_run(net, m0, shadow, ids, y, False)
    emu = fp64_run(net, m0, shadow, ids, y, True)
    grad = net.spec.views(flat)
    items = [("loss", loss.detach().double().reshape(()), f64[0], emu[0])]
    items += [(e.name, grad[e.name].double(), f64[1][e.name], emu[1][e.name]) for e in net.spec.entries]
    bad, report = [], []
    for name, k, ref, em in items:
        ek = float((k - ref.reshape(k.shape)).norm())
        ee = float((em.reshape(k.shape) - ref.reshape(k.shape)).norm())
        rn = float(ref.norm())
        floor = (BF_U if k.numel() == 1 else 2.0 ** -16) * rn + 1e-30
        report.append(f"{name}: {ek / ee if ee else 0:.2f}")
        if k.numel() > 1 and rn < ee:                 # zero in exact arithmetic: the key biases
            continue
        if not math.isfinite(ek) or ek > RATIO * ee + floor:
            bad.append(f"{name}: ||kernel - fp64|| {ek:.3g} > {RATIO} x ||emulation - fp64|| {ee:.3g} + {floor:.3g}")
    print("GPT e2e ratios:", ", ".join(report))
    assert not bad, "; ".join(bad)
    # the tied head's contribution is there: the word gradient is not just the embedding scatter
    assert float(grad["emb.word"][~torch.isin(torch.arange(SMALL["vocab"], device="cuda"),
                                             ids.long().unique())].abs().sum()) > 0


# ------------------------------------------------------------------------------ stages
def _rows_of(t):
    return t.double().reshape(-1, t.shape[-1])


def stage_embedding(run, r, S):
    ids = r["hp"]["ids"].long()
    table, pos = r["pv"]["table"], r["pv"]["pos"]
    pid = torch.arange(ids.numel(), device="cuda") % S
    ref = table[ids] + pos[pid]
    MC._assert("stage", r["out"], ref, U * ref.abs(), "embedding output")
    dy = r["dy"].double()
    gp = MC.grad_view(run, "emb.pos")
    want = torch.zeros(gp.shape, dtype=F64, device="cuda").index_add_(0, pid, dy)
    cnt = torch.zeros(gp.shape[0], 1, dtype=F64, device="cuda").index_add_(0, pid, torch.ones_like(dy[:, :1]))
    sl = MC.gam(1) * cnt * torch.zeros(gp.shape, dtype=F64, device="cuda").index_add_(0, pid, dy.abs())
    MC._assert("stage", gp, want, sl, "embedding position gradient")
    return ids, dy


def stage_attention_causal(r):
    hp = r["hp"]
    B, S, H = hp["B"], hp["S"], hp["H"]
    assert hp["causal"] and hp["lengths"] is None
    lay = lambda t: MC._heads(t, B, S, H)  # noqa: E731
    q, k, v = (lay(r["in"][x]) for x in ("q", "k", "v"))
    mask = causal_mask(B * H, S).to("cuda")
    o = lay(r["out"])
    rf = causal_ref_fwd(q, k, v, mask, 0.125)
    fb = causal_fwd_bounds(q, k, v, mask, 0.125, rf)
    assert not attn_violations(o, rf["o"], fb["o"]).any(), f"{r['id']} output out of bound"
    if r["dy"] is None:
        return
    lse = r["lse"][:B * H * S].view(B * H, S).double()
    do = lay(r["dy"])
    rb = causal_ref_bwd(q, k, v, do, o, lse, mask, 0.125)
    bb = causal_bwd_bounds(q, k, v, do, o, lse, mask, 0.125, rb)
    for x in ("q", "k", "v"):
        n = int(attn_violations(lay(r["dx"][x]), rb["d" + x], bb["d" + x]).sum())
        assert n == 0, f"{r['id']} d{x}: {n} elements out of bound"


def stage_lm_head(run, r, emb):
    """Loss, dh and the tied word gradient = embedding scatter + dlogits^T h."""
    h = r["in"]["h"].double()
    w = run["net"].spec.views(run["shadow"])["emb.word"].double()
    t = r["hp"]["targets"].long()
    M, K = h.shape
    z = h @ w.t()
    ez = MC.gam(K) * (h.abs() @ w.abs().t())               # fp32 logits of exact bf16 products
    loss_rows, g, lb, _ = xent_bounds(z.cpu(), t.cpu(), 1.0 / M)
    shift = 2 * ez.amax(-1).cpu()                           # the logits' error moves lse and z_t
    err = abs(float(r["out"]) - float(loss_rows.mean()))
    assert err <= float((lb + shift).mean()) + MC.gam(M) * float(loss_rows.abs().mean()), f"head loss: {err}"
    g = g.cuda()
    p = torch.softmax(z, -1)
    onehot = TF.one_hot(t, w.shape[0]).to(F64)
    e_dl = (p * (torch.exp(2 * ez.amax(-1, keepdim=True)) - 1) + 2 * BF_U * (p + onehot) + 1e-7) / M
    adl = g.abs() + e_dl
    MC._assert("stage", r["dx"]["h"], g @ w, e_dl @ w.abs() + MC.gam(w.shape[0] + 64) * (adl @ w.abs()), "head dh")
    ids, dy = emb
    gw = MC.grad_view(run, "emb.word")
    scatter = torch.zeros(gw.shape, dtype=F64, device="cuda").index_add_(0, ids, dy)
    sabs = torch.zeros(gw.shape, dtype=F64, device="cuda").index_add_(0, ids, dy.abs())
    head = g.t() @ h
    sl = e_dl.t() @ h.abs() + MC.gam(M + 64) * (adl.t() @ h.abs()) + 2 * MC.gam(M + 2) * (sabs + head.abs())
    MC._assert("stage", gw, scatter + head, sl, "tied emb.word gradient (scatter + head)")


def test_gpt_stage_by_stage(monkeypatch):
    """One training step under the model-conformance recorder, every op checked from its own operands."""
    monkeypatch.setitem(MC.ACTS, "lm_xent", ("h",))
    net, b, master, shadow, grad = make()
    ids, y = data(B=2)
    with MC.Recorder(monkeypatch, net.spec, {"P": master, "S": shadow, "G": grad}) as rec:
        loss = net.loss(b, ids, y)
        loss.backward()
    torch.cuda.synchronize()
    run = dict(net=net, grad=grad, master=master, shadow=shadow)
    ops = [r["op"] for r in rec.calls]
    L = net.L
    assert ops.count("linear") == 6 * L and ops.count("layernorm") == 2 * L + 1 and ops.count("add") == 2 * L
    assert ops.count("attention") == L and ops.count("embedding") == 1 and ops[-1] == "lm_xent", ops
    emb = None
    for i, r in enumerate(rec.calls):
        r["id"] = f"{r['op']}#{i}"
        op = r["op"]
        if op == "linear":
            MC.stage_linear(run, r, False)
        elif op == "layernorm":
            MC.stage_ln(run, r)
        elif op == "add":
            MC.stage_add(run, r)
        elif op == "embedding":
            emb = stage_embedding(run, r, ids.shape[1])
        elif op == "attention":
            stage_attention_causal(r)
        elif op == "lm_xent":
            stage_lm_head(run, r, emb)
        else:
            raise AssertionError(f"unexpected op {op}")


def test_gpt_causal_through_the_model():
    net, b, _, _, _ = make()
    ids, _ = data(B=2, S=128)
    S = ids.shape[1]
    h0 = net.features(b, ids, False).view(2, S, -1)
    for t in (0, 63, 64, 100, 127):
        ids2 = ids.clone()
        ids2[:, t] = (ids2[:, t] + 1) % SMALL["vocab"]
        h1 = net.features(b, ids2, False).view(2, S, -1)
        assert torch.equal(h0[:, :t].view(torch.int16), h1[:, :t].view(torch.int16)), t
        assert not torch.equal(h0[:, t], h1[:, t]), t


def test_gpt_dropout_sites_and_masks(monkeypatch):
    import inspect
    from bflc_demo_b200._native import C
    from bflc_demo_b200.ops import nn as NN
    from bflc_demo_b200.ops.nn import DropoutRNG
    net, b, _, _, _ = make(dropout=0.1)
    ids, y = data()
    step = torch.tensor([3], device="cuda", dtype=torch.int32)
    seen, depth = [], [0]

    def spy(op):
        fn, sig = getattr(NN, op), inspect.signature(getattr(NN, op))

        def wrapper(*a, **kw):
            if depth[0] == 0:                        # the model's calls only (dropout calls dropout_add)
                ba = sig.bind(*a, **kw)
                ba.apply_defaults()
                p = ba.arguments.get("dropout_p", ba.arguments.get("p"))
                seen.append((op, int(ba.arguments["site"]), float(p)))
            depth[0] += 1
            try:
                return fn(*a, **kw)
            finally:
                depth[0] -= 1
        monkeypatch.setattr(NN, op, wrapper)

    for op in ("dropout", "dropout_add", "attention"):
        spy(op)
    l1 = net.loss(b, ids, y, rng=DropoutRNG(7, step, 0)).detach()
    want = [("dropout", 0, 0.1)]
    for i in range(net.L):
        want += [("attention", 8 * i + 1, 0.1), ("dropout_add", 8 * i + 2, 0.1), ("dropout_add", 8 * i + 3, 0.1)]
    assert seen == want, seen
    monkeypatch.undo()
    l2 = net.loss(b, ids, y, rng=DropoutRNG(7, step, 0)).detach()
    l3 = net.loss(b, ids, y, rng=DropoutRNG(7, step, 1)).detach()
    assert torch.equal(l1, l2) and not torch.equal(l1, l3)
    with pytest.raises(ValueError):
        net.loss(b, ids, y)                       # dropout > 0 needs an rng
    assert torch.equal(net.correct(b, ids, y), net.correct(b, ids, y))   # never drops
    # every site draws its own mask: attention keep masks and hidden masks
    sites = sorted({s for _, s, _ in want})
    masks = []
    for site in sites:
        m = torch.empty(2 * 2 * 64 * 64, device="cuda", dtype=torch.uint8)
        C().dropout_keep_mask(m, 2, 2, 64, 0.1, 7, step, 0, site)
        h = NN.dropout(torch.ones(128, 64, device="cuda", dtype=BF16), 0.1, DropoutRNG(7, step, 0), site, S=64)
        masks.append((m, h))
    for i in range(len(sites)):
        for j in range(i + 1, len(sites)):
            assert not torch.equal(masks[i][0], masks[j][0]) and not torch.equal(masks[i][1], masks[j][1]), \
                (sites[i], sites[j])


def test_gpt_correct_matches_fp64_argmax():
    """Targets: the fp64 argmax on every other clear-margin row, the least likely token on all other
    rows, so the fp64 count is exact and a ``correct`` that drops or invents hits fails."""
    net, b, master, shadow, _ = make()
    ids, _ = data(B=8)
    h = net.features(b, ids, False)                  # the forward is deterministic: correct() sees this h
    w = net.spec.views(shadow)["emb.word"]
    z = h.double() @ w.double().T
    ez = MC.gam(h.shape[1]) * (h.double().abs() @ w.double().abs().T).amax(-1)
    top = z.topk(2, -1).values
    clear = (top[:, 0] - top[:, 1]) > 2 * ez
    pick = clear & (torch.arange(z.shape[0], device="cuda") % 2 == 0)
    t = torch.where(pick, z.argmax(-1), z.argmin(-1)).to(torch.int32)
    assert int(pick.sum()) > z.shape[0] // 4
    assert int(net.correct(b, ids, t.view(ids.shape))) == int(pick.sum())


def _engine(capture, rounds, lr=2e-3):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import lm_corpus_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import GPT
    cfg = FLConfig.for_world(1, model="gpt", batch_size=16, samples_per_client=64, learning_rate=2e-3,
                             optimizer="adam", cuda_graph=capture, val_samples=32)
    shard = lm_corpus_like(1, 64, seed=3, seq_len=128, vocab=512, only=0)[0]
    eng = GenericFedEngine(cfg, GPT(**SMALL), shard, rank=0, world=1, device=0)
    eng.cfg.learning_rate = lr                      # 0: frozen weights (the config itself insists on lr > 0)
    if capture:
        eng.capture()
    for _ in range(rounds):
        eng.run_round()
    return eng, shard


def test_gpt_captured_training_pass_equals_eager_bit_for_bit():
    """lr = 0: the weights never move, so the training pass's loss (the forward of every step) is a
    deterministic function of the state: one replay of the captured pass and one eager pass agree
    bit for bit."""
    eng, _ = _engine(True, 0, lr=0.0)
    assert eng.capture_error == "" and eng.graph_train is not None
    m0 = eng.work_master.clone()

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
    assert torch.equal(eng.work_master, m0)


def test_gpt_engine_rounds_scores_and_learning():
    from bflc_demo_b200.data.synthetic import lm_corpus_like
    test = lm_corpus_like(1, 32, seed=3, seq_len=128, vocab=512, only=0)[0]
    a, shard = _engine(True, 3)
    b, _ = _engine(False, 4)             # capture() runs one eager round first: 4 rounds each
    c, _ = _engine(False, 4)
    assert a.capture_error == "" and a.graph_train is not None
    torch.cuda.synchronize()
    # whole trained rounds: within the spread of two eager runs (fp32 atomics in the embedding backward)
    d_graph = float((a.global_master - b.global_master).abs().max())
    d_eager = float((c.global_master - b.global_master).abs().max())
    print(f"GPT engine: |graph - eager| {d_graph:.3g}, |eager - eager| {d_eager:.3g}")
    assert d_graph <= max(4 * d_eager, 1e-6), (d_graph, d_eager)
    for eng in (a, b, c):
        assert eng.drain_blocks() == [] and eng.host_ledger.verify_chain()
    from bflc_demo_b200.engine.base import parse_block_record
    assert a.n_val_targets == 32 * 128
    hits = int(a.val_correct[0])                     # the last round's committee count
    ring, size = a.ring_bytes.cpu().numpy(), a.sz["BlockRecord"]
    recs = [parse_block_record(ring, slot * size, 1) for slot in range(8)]
    last = max(recs, key=lambda r: r[0])[2]
    score = float(last["score_rows"][0][0])
    assert 0.0 <= score <= 1.0
    assert abs(score - hits / (32 * 128)) <= 1e-6, (score, hits)
    acc0 = b.evaluate(test)
    for _ in range(8):
        b.run_round()
    acc = b.evaluate(test)
    print(f"GPT next-token test accuracy {acc0:.4f} -> {acc:.4f} after 12 rounds")
    # chance is 1 / 512 = 0.0020; measured 0.0029 -> 0.0088 on an H100 80GB HBM3 at a 700 W power limit
    assert acc > 3 / 512 and acc > acc0, (acc0, acc)
