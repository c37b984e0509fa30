"""Block-scaled fp8 (MXFP8) flagship path: input preparation, weight blobs, the persistent
trainer with fwd1/fwd2 on block-scaled e4m3 wgmma and its fused
UploadLocalUpdate, and the fp8 committee validation -- each against plain PyTorch.

The trainer is checked on parameter DELTAS (w_after - w_before), not on weights: one SGD step
moves a weight by O(1e-2) of its norm, so a weight-level tolerance would pass a badly scaled
gradient.  Two oracles: (a) an fp32 PyTorch emulation of the exact recipe (same quantisation
points, bf16 where the kernel uses bf16) -> tight tolerance, catches a wrong scale byte / tile;
(b) plain fp32 autograd of the unquantised model -> loose tolerance, bounds the fp8 noise."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel(x, ref):
    return ((x.float() - ref.float()).norm() / (ref.float().norm() + 1e-12)).item()


def q_dq(x):
    """fp32 [R, K] -> dequantised MXFP8 (e4m3 + one power-of-two scale per 32 K-elements)."""
    from bflc_demo_b200.ops.mx8 import quantize_mx8_reference
    return quantize_mx8_reference(x.float()).dequantize()


def bf(x):
    return x.to(torch.bfloat16).float()


def emulate_steps(init, spec, xu8, y, B, steps, lr, adam=False):
    """fp32 PyTorch emulation of the persistent trainer's fp8 recipe (csrc/kernels/mlp_round_sm100.cu)."""
    p = {k: v.clone().float() for k, v in spec.views(init.clone()).items()}
    m = {k: torch.zeros_like(v) for k, v in p.items()}
    v2 = {k: torch.zeros_like(v) for k, v in p.items()}
    xf = xu8.float() / 255.0
    loss_sum = 0.0
    for s in range(steps):
        xb, yb = xf[s * B:(s + 1) * B], y[s * B:(s + 1) * B].long()
        xq = q_dq(xb)
        h = torch.relu(xq @ q_dq(p["w1"]).t() + p["b1"])
        hq = q_dq(h)
        logits = hq @ q_dq(p["w2"]).t() + p["b2"]
        loss_sum += torch.nn.functional.cross_entropy(logits, yb, reduction="sum").item()
        dl = (torch.softmax(logits, -1) - torch.nn.functional.one_hot(yb, logits.shape[1]).float()) / B
        dl_b, h_b, x_b = bf(dl), bf(h), bf(xb)
        dh = (dl_b @ bf(p["w2"])) * (hq > 0).float()
        g = {"w2": dl_b.t() @ h_b, "b2": dl.sum(0), "w1": bf(dh).t() @ x_b, "b1": dh.sum(0)}
        for k in p:
            if adam:
                t = s + 1
                m[k] = 0.9 * m[k] + 0.1 * g[k]
                v2[k] = 0.999 * v2[k] + 0.001 * g[k] * g[k]
                p[k] = p[k] - lr * (m[k] / (1 - 0.9 ** t)) / ((v2[k] / (1 - 0.999 ** t)).sqrt() + 1e-8)
            else:
                p[k] = p[k] - lr * g[k]
    return p, loss_sum


def autograd_steps(init, spec, xu8, y, B, steps, lr):
    p = {k: v.clone().float().requires_grad_(True) for k, v in spec.views(init.clone()).items()}
    xf = xu8.float() / 255.0
    for s in range(steps):
        xb, yb = xf[s * B:(s + 1) * B], y[s * B:(s + 1) * B].long()
        loss = torch.nn.functional.cross_entropy(torch.relu(xb @ p["w1"].t() + p["b1"]) @ p["w2"].t() + p["b2"], yb)
        gr = torch.autograd.grad(loss, list(p.values()))
        p = {k: (v - lr * g).detach().requires_grad_(True) for (k, v), g in zip(p.items(), gr)}
    return {k: v.detach() for k, v in p.items()}


def test_prep_inputs_bf16_and_mx8():
    from bflc_demo_b200._native import C
    from bflc_demo_b200.models.mlp import sf_bytes
    from bflc_demo_b200.ops.mx8 import MX8, quantize_mx8_reference
    torch.manual_seed(0)
    R, K = 512, 784
    x = torch.randint(0, 256, (R, K), device="cuda", dtype=torch.uint8)
    x[:, 300:340] = 0                                   # an all-zero group: scale 1.0, zeros
    xb = torch.empty(R, K, device="cuda", dtype=torch.bfloat16)
    xq = torch.zeros(R, K, device="cuda", dtype=torch.uint8)
    xsf = torch.full((sf_bytes(R, K),), 127, device="cuda", dtype=torch.uint8)
    C().prep_inputs(x, xb, xq, xsf, 1.0 / 255.0)
    torch.cuda.synchronize()
    assert torch.equal(xb, (x.float() * (1.0 / 255.0)).to(torch.bfloat16))
    ref = quantize_mx8_reference(x.float() * (1.0 / 255.0))
    got = MX8(xq.view(torch.float8_e4m3fn), xsf, R, K)
    assert torch.equal(got.dequantize(), ref.dequantize())
    # the K-tail group (16 valid columns) and the padding groups of the last K-block
    kb = (K + 127) // 128
    sf = xsf.view(R // 128, kb, 32, 4, 4)
    assert int(sf[:, kb - 1, :, :, 1:].min()) == 127 and int(sf[:, kb - 1, :, :, 1:].max()) == 127
    assert rel(got.dequantize(), x.float() / 255.0) < 0.04


def test_quantize_mlp_blob_layout():
    from bflc_demo_b200._native import C
    from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec
    from bflc_demo_b200.ops.mx8 import MX8
    spec = mlp_spec(784, 256, 62)
    init = torch.empty(spec.total)
    spec.init_(init, seed=3)
    master = init.cuda()
    tr = FlatMLP(spec, master, master.bfloat16(), torch.zeros_like(master), 512, fp8=True)
    blob = tr.quantize_weights()
    torch.cuda.synchronize()
    L, p = tr.ql, spec.views(master)
    w1 = MX8(blob[L["w1q"]:L["w1q"] + 256 * 784].view(256, 784).view(torch.float8_e4m3fn),
             blob[L["w1sf"]:L["w1sf"] + 2 * L["kb1"] * 512], 256, 784)
    assert torch.equal(w1.dequantize(), q_dq(p["w1"]))
    w2 = MX8(blob[L["w2q"]:L["w2q"] + 64 * 256].view(64, 256).view(torch.float8_e4m3fn),
             blob[L["w2sf"]:L["w2sf"] + L["kb2"] * 512], 64, 256)
    d2 = w2.dequantize()
    assert torch.equal(d2[:62], q_dq(p["w2"])) and float(d2[62:].abs().max()) == 0.0
    b1 = blob[L["b1"]:L["b1"] + 1024].view(torch.float32)
    b2 = blob[L["b2"]:L["b2"] + 256].view(torch.float32)
    assert torch.equal(b1, p["b1"]) and torch.equal(b2[:62], p["b2"]) and float(b2[62:].abs().max()) == 0.0
    assert C().mx8_mlp_layout(784, 256)["total"] == L["total"]


def _fp8_trainer(init, spec, B, opt, lr):
    from bflc_demo_b200.models.mlp import FlatMLP
    master = init.cuda().clone()
    tr = FlatMLP(spec, master, master.bfloat16(), torch.zeros_like(master), B, lr=lr, optimizer=opt, fp8=True)
    tr.quantize_weights()
    return tr, master


def _prep(xu8):
    from bflc_demo_b200._native import C
    from bflc_demo_b200.models.mlp import sf_bytes
    R, K = xu8.shape
    xb = torch.empty(R, K, device="cuda", dtype=torch.bfloat16)
    xq = torch.zeros(R, K, device="cuda", dtype=torch.uint8)
    xsf = torch.full((sf_bytes(R, K),), 127, device="cuda", dtype=torch.uint8)
    C().prep_inputs(xu8, xb, xq, xsf, 1.0 / 255.0)
    return xb, xq, xsf


@pytest.mark.parametrize("B,steps,opt,lr", [(512, 1, "sgd", 0.05), (512, 4, "sgd", 0.05), (256, 3, "adam", 1e-3),
                                            (128, 2, "sgd", 0.1)])
def test_fp8_trainer_deltas_vs_emulation_and_autograd(B, steps, opt, lr):
    from bflc_demo_b200.models.mlp import mlp_spec
    torch.manual_seed(5)
    spec = mlp_spec(784, 256, 62)
    init = torch.empty(spec.total)
    spec.init_(init, seed=2)
    xu8 = (torch.rand(B * steps, 784, device="cuda") ** 2 * 255).to(torch.uint8)
    y = torch.randint(0, 62, (B * steps,), device="cuda", dtype=torch.int32)
    xb, xq, xsf = _prep(xu8)
    tr, master = _fp8_trainer(init, spec, B, opt, lr)
    bar = torch.zeros(1, device="cuda", dtype=torch.int32)
    tr.train_epoch_fused(xb, y, steps, bar.data_ptr(), None, 3, 1, x_q=xq, x_sf=xsf)
    torch.cuda.synchronize()
    w0 = spec.views(init.cuda())
    got = {k: v - w0[k] for k, v in spec.views(master).items()}
    emu, loss_emu = emulate_steps(init.cuda(), spec, xu8, y, B, steps, lr, adam=opt == "adam")
    for k in ("w1", "b1", "w2", "b2"):
        assert rel(got[k], emu[k] - w0[k]) < (2e-2 if opt == "sgd" else 0.15), (k, rel(got[k], emu[k] - w0[k]))
    assert abs(tr.loss_sum.item() - loss_emu) / loss_emu < 5e-3
    if opt == "sgd":
        ref = autograd_steps(init.cuda(), spec, xu8, y, B, steps, lr)
        for k in ("w1", "w2"):
            assert rel(got[k], ref[k] - w0[k]) < 0.25, (k, rel(got[k], ref[k] - w0[k]))
    # the compute copies were refreshed by the optimizer epilogue: bf16 shadow and the MXFP8 blob
    from bflc_demo_b200.ops.mx8 import MX8
    p, L, blob = spec.views(master), tr.ql, tr.work_q
    assert rel(tr.shadow.float(), master) < 4e-3
    w1 = MX8(blob[L["w1q"]:L["w1q"] + 256 * 784].view(256, 784).view(torch.float8_e4m3fn),
             blob[L["w1sf"]:L["w1sf"] + 2 * L["kb1"] * 512], 256, 784)
    w2 = MX8(blob[L["w2q"]:L["w2q"] + 64 * 256].view(64, 256).view(torch.float8_e4m3fn),
             blob[L["w2sf"]:L["w2sf"] + L["kb2"] * 512], 64, 256)
    assert torch.equal(w1.dequantize(), q_dq(p["w1"]))
    assert torch.equal(w2.dequantize()[:62], q_dq(p["w2"]))


def test_fp8_ranking_matches_bf16():
    """The committee's score ORDER is the protocol's security mechanism (SURVEY.md 7.5.7): models of
    clearly different quality must rank the same under fp8 and bf16 validation."""
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    accs = {}
    for dt in ("bf16", "fp8"):
        cfg = FLConfig.for_world(1, model="mlp", hidden=256, batch_size=512, samples_per_client=2048,
                                 learning_rate=0.05, dtype=dt, cuda_graph=False)
        eng = FusedEngine(cfg, femnist_like(1, 2048, seed=7, only=0)[0])
        test = femnist_like(2, 2048, seed=7, only=1)[0]      # same class prototypes, unseen samples
        a = [eng.evaluate(test)]
        for _ in range(10):
            eng.run_round()
            a.append(eng.evaluate(test))
        assert not eng.drain_blocks()
        accs[dt] = a
        del eng
    # both learn (held-out accuracy far above the 1/62 prior), and the two curves stay close
    for dt in accs:
        assert accs[dt][-1] > accs[dt][0] + 0.3, accs
    assert all(abs(a - b) < 0.05 for a, b in zip(accs["bf16"], accs["fp8"])), accs


@pytest.mark.parametrize("dtype,optimizer", [("fp8", "sgd"), ("fp8", "adam"), ("bf16", "sgd")])
def test_fused_upload_publishes_what_was_trained(dtype, optimizer):
    """The trainer's last optimizer epilogue is UploadLocalUpdate: in a solo round FedAvg has one
    operand with weight 1, so the new global model must equal the uploaded fp32 weights bit for
    bit, the upload must be a real training result (!= genesis) and the fp8 blob must be the
    quantisation of exactly those weights."""
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    from bflc_demo_b200.ops.mx8 import MX8
    cfg = FLConfig.for_world(1, model="mlp", hidden=256, batch_size=512, samples_per_client=2048,
                             learning_rate=0.05 if optimizer == "sgd" else 1e-3, dtype=dtype,
                             optimizer=optimizer, cuda_graph=True)
    eng = FusedEngine(cfg, femnist_like(1, 2048, seed=7, only=0)[0])
    assert eng.fused_upload
    genesis = eng.global_master.clone()
    eng.capture()                      # runs round 0 eagerly
    eng.run_round()                    # round 1 from the graph
    torch.cuda.synchronize()
    st = eng.read_state()
    assert st["epoch"] == 2 and not eng.drain_blocks()
    par = (st["epoch"] - 1) & 1
    o, P = eng.layout.offsets, eng.n_params
    up = eng.heap.view(o[f"upload_master{par}"], [P], torch.float32)
    assert torch.equal(up, eng.global_master)
    assert rel(up, genesis) > 1e-3
    sp = eng.spec.views(up)
    if dtype == "fp8":
        L = eng.ql
        blob = eng.heap.view(eng.upq_off[par], [eng.blob_bytes], torch.uint8)
        w1 = MX8(blob[L["w1q"]:L["w1q"] + 256 * 784].view(256, 784).view(torch.float8_e4m3fn),
                 blob[L["w1sf"]:L["w1sf"] + 2 * L["kb1"] * 512], 256, 784)
        assert torch.equal(w1.dequantize(), q_dq(sp["w1"]))
        assert torch.equal(blob[L["b1"]:L["b1"] + 1024].view(torch.float32), sp["b1"])
        assert torch.equal(blob[L["b2"]:L["b2"] + 248].view(torch.float32), sp["b2"])
    else:
        sh = eng.heap.view(o[f"upload_shadow{par}"], [P], torch.bfloat16)
        assert torch.equal(sh, up.to(torch.bfloat16))
    assert 0.0 < st["global_loss"] < 4.2     # mean xent of the local pass (ln 62 = 4.13 at init)


def test_mlp_val_fp8_counts():
    """fp8 committee validation (one launch per committee member) vs the PyTorch emulation."""
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    cfg = FLConfig.for_world(1, model="mlp", hidden=256, batch_size=512, samples_per_client=2048,
                             learning_rate=0.05, dtype="fp8", cuda_graph=False)
    shard = femnist_like(1, 2048, seed=7, only=0)[0]
    eng = FusedEngine(cfg, shard)
    eng.run_round()
    eng.run_round()
    torch.cuda.synchronize()
    st = eng.read_state()
    par = (st["epoch"] - 1) & 1
    up = eng.heap.view(eng.layout.offsets[f"upload_master{par}"], [eng.n_params], torch.float32)
    p = eng.spec.views(up)
    x = shard.x.reshape(len(shard), -1).cuda().float() / 255.0
    h = torch.relu(q_dq(x) @ q_dq(p["w1"]).t() + p["b1"])
    pred = (q_dq(h) @ q_dq(p["w2"]).t() + p["b2"]).argmax(-1)
    want = int((pred == shard.y.cuda()).sum())
    got = int(eng.val_correct[0].item())
    assert abs(got - want) <= 0.01 * len(shard), (got, want)
    assert abs(st["median"][0] - got / len(shard)) < 1e-6
