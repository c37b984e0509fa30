"""The fp8 trainer and the fp8 committee validation run bf16 wgmma on exactly dequantised MXFP8
copies: every copy must equal ``quantize_mx8_reference(...).dequantize()`` bit for bit, and the
trainer must track the fp32 emulation of the recipe more tightly than the e4m3-accumulating
mainloop it replaced."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest
import torch

from bflc_demo_b200 import build


def _dq_ref(x):
    from bflc_demo_b200.ops.mx8 import quantize_mx8_reference
    return quantize_mx8_reference(x.float()).dequantize()


def fp8_gmma_lines(src, root):
    """SASS lines of `src` (compiled exactly as the build compiles it, includes under `root`) that
    issue an fp8 wgmma: on sm_90a those disassemble as QGMMA (bf16 / f16 ones as HGMMA)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, "k.o")
        inc = [f"-I{os.path.join(root, d)}" for d in ("include", "ledger", "runtime")]
        subprocess.run([nvcc, *build.GENCODE, *build.NVCC_FLAGS, *inc, "-c", str(src), "-o", obj],
                       check=True, capture_output=True, timeout=900)
        sass = subprocess.run([cuobjdump, "-sass", obj], check=True, capture_output=True, text=True).stdout
    gmma = [ln for ln in sass.splitlines() if "GMMA" in ln]
    assert gmma, "no wgmma at all: the disassembly format changed"
    return [ln for ln in gmma if "QGMMA" in ln or re.search(r"E4M3|E5M2", ln)]


@pytest.mark.parametrize("kernel", ["mlp_round_sm100.cu", "mlp_val_sm100.cu"])
def test_no_fp8_wgmma_in_trainer_or_validation(kernel):
    """CPU: the persistent trainer (both instantiations) and the committee validation kernel
    multiply MXFP8 operands as bf16 wgmma; no e4m3 wgmma may come back."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if shutil.which(nvcc) is None or not os.path.exists(os.path.join(os.path.dirname(nvcc), "cuobjdump")):
        pytest.skip("no CUDA toolkit")
    bad = fp8_gmma_lines(build.CSRC / "kernels" / kernel, build.CSRC)
    assert not bad, "\n".join(bad[:4])


gpu = pytest.mark.gpu


def _prep(xu8):
    from bflc_demo_b200._native import C
    from bflc_demo_b200.models.mlp import sf_bytes
    R, K = xu8.shape
    xb = torch.empty(R, K, device="cuda", dtype=torch.bfloat16)
    xq = torch.zeros(R, K, device="cuda", dtype=torch.uint8)
    xsf = torch.full((sf_bytes(R, K),), 127, device="cuda", dtype=torch.uint8)
    xdq = torch.empty(R, K, device="cuda", dtype=torch.bfloat16)
    C().prep_inputs(xu8, xb, xq, xsf, 1.0 / 255.0, xdq)
    return xb, xq, xsf, xdq


@gpu
def test_x_dq_from_both_prep_kernels():
    from bflc_demo_b200._native import C
    torch.manual_seed(0)
    R, K = 512, 784
    x = torch.randint(0, 256, (R, K), device="cuda", dtype=torch.uint8)
    x[:, 300:340] = 0
    _, xq, xsf, xdq = _prep(x)
    torch.cuda.synchronize()
    ref = _dq_ref(x.float() / 255.0)
    assert torch.equal(xdq.float(), ref)
    # the derived copy (x_q + x_sf only) is the same
    d2 = torch.empty_like(xdq)
    C().mx8_dequant(xq, xsf, d2)
    # the chunked (input pipeline) kernel: tags already match the device round counter
    steps, rows = 4, R // 4
    flags = torch.ones(16, device="cuda", dtype=torch.int32)
    seq = torch.zeros(1, device="cuda", dtype=torch.int32)
    cnt = torch.zeros(16, device="cuda", dtype=torch.int32)
    ready = torch.zeros(16, device="cuda", dtype=torch.int32)
    err = torch.zeros(1, device="cuda", dtype=torch.int32)
    d3 = torch.empty_like(xdq)
    C().prep_inputs_chunks(x, None, None, None, rows, steps, 1.0 / 255.0, flags, seq, cnt, ready, err, d3)
    torch.cuda.synchronize()
    assert torch.equal(d2, xdq) and torch.equal(d3, xdq) and int(err.item()) == 0


@gpu
def test_smallest_scale_groups_are_exact():
    """Groups at the smallest scale byte the quantisers emit (3): one whose amax sets it exactly,
    with e4m3 values below 0.25 whose products are bf16 subnormals, and one whose amax asks for a
    smaller byte and is clamped up to 3."""
    from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec
    from bflc_demo_b200.ops.mx8 import MX8
    spec = mlp_spec(784, 256, 62)
    master = torch.zeros(spec.total, device="cuda")
    w1 = spec.views(master)["w1"]
    # amax = 448 * 2^-124 -> byte 3 (inputs stay normal fp32 values: the fast-math quantisers flush
    # smaller ones, so the bf16-subnormal products of this scale are checked on raw codes below)
    g = torch.tensor([448.0, 1.0, 0.25, 0.375, -0.5, 0.3, 0.0, 240.0] * 4)
    w1[5, 64:96] = (g * 2.0 ** -124).cuda()
    # amax = 2^-125: the formula asks for byte 127 + ceil(log2(2^-125 / 448)) = 127 - 133 < 3
    w1[9, 0:32] = 2.0 ** -125
    tr = FlatMLP(spec, master, master.bfloat16(), torch.zeros_like(master), 128, fp8=True)
    tr.quantize_weights()
    torch.cuda.synchronize()
    L = tr.ql
    sf = tr.work_q[L["w1sf"]:L["w1sf"] + 2 * L["kb1"] * 512]
    chunk = sf.view(2, L["kb1"], 32, 4, 4)
    assert int(chunk[0, 0, 5, 0, 2]) == 3 and int(chunk[0, 0, 9, 0, 0]) == 3
    want = _dq_ref(spec.views(master)["w1"])
    got = tr.work_dq[:256 * 784].view(256, 784).float()
    assert torch.equal(got, want)
    assert float(got[5, 64]) == 448.0 * 2.0 ** -124 and float(got[9, 0]) == 2.0 ** -125
    # every e4m3 code at scale byte 3, through the dequantise kernel: bf16 subnormals down to 2^-133
    from bflc_demo_b200._native import C
    codes = torch.arange(256, dtype=torch.int32)
    codes = codes[(codes & 0x7F) != 0x7F].to(torch.uint8)           # drop the two NaN codes
    q = torch.zeros(128, 256, dtype=torch.uint8)
    q[0, :codes.numel()] = codes
    sfb = torch.full((1 * 2 * 512,), 127, dtype=torch.uint8)
    for grp in range(8):
        sfb[(grp // 4) * 512 + grp % 4] = 3                          # row 0, K-groups 0..7
    d = torch.empty(128, 256, dtype=torch.bfloat16, device="cuda")
    C().mx8_dequant(q.cuda(), sfb.cuda(), d)
    ref = MX8(q.view(torch.float8_e4m3fn), sfb, 128, 256).dequantize()
    assert torch.equal(d.float().cpu(), ref)
    assert float(d[0, 1]) == 2.0 ** -133                           # the smallest e4m3 subnormal


def _blob_dq(blob, L):
    from bflc_demo_b200.ops.mx8 import MX8
    w1 = MX8(blob[L["w1q"]:L["w1q"] + 256 * 784].view(256, 784).view(torch.float8_e4m3fn),
             blob[L["w1sf"]:L["w1sf"] + 2 * L["kb1"] * 512], 256, 784)
    w2 = MX8(blob[L["w2q"]:L["w2q"] + 64 * 256].view(64, 256).view(torch.float8_e4m3fn),
             blob[L["w2sf"]:L["w2sf"] + L["kb2"] * 512], 64, 256)
    return w1.dequantize(), w2.dequantize()


@gpu
@pytest.mark.parametrize("opt,lr,steps", [("sgd", 0.05, 4), ("adam", 1e-3, 3)])
def test_work_dq_and_trainer_vs_emulation(opt, lr, steps):
    from test_gpu_mlp_fp8 import emulate_steps, rel
    from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec
    torch.manual_seed(5)
    B = 256
    spec = mlp_spec(784, 256, 62)
    init = torch.empty(spec.total)
    spec.init_(init, seed=2)
    master = init.cuda().clone()
    tr = FlatMLP(spec, master, master.bfloat16(), torch.zeros_like(master), B, lr=lr, optimizer=opt, fp8=True)
    tr.quantize_weights()
    torch.cuda.synchronize()
    p = spec.views(master)
    d1, d2 = tr.work_dq[:256 * 784].view(256, 784), tr.work_dq[256 * 784:].view(64, 256)
    assert torch.equal(d1.float(), _dq_ref(p["w1"])) and torch.equal(d2[:62].float(), _dq_ref(p["w2"]))
    assert float(d2[62:].float().abs().max()) == 0.0
    xu8 = (torch.rand(B * steps, 784, device="cuda") ** 2 * 255).to(torch.uint8)
    y = torch.randint(0, 62, (B * steps,), device="cuda", dtype=torch.int32)
    xb, _, _, xdq = _prep(xu8)
    bar = torch.zeros(1, device="cuda", dtype=torch.int32)
    tr.train_epoch_fused(xb, y, steps, bar.data_ptr(), None, 3, 1, x_dq=xdq)
    torch.cuda.synchronize()
    # after training: work_dq == dequantised blob == dequantised master
    b1, b2 = _blob_dq(tr.work_q, tr.ql)
    assert torch.equal(d1.float(), b1) and torch.equal(d1.float(), _dq_ref(p["w1"]))
    assert torch.equal(d2.float(), b2) and torch.equal(d2[:62].float(), _dq_ref(p["w2"]))
    w0 = spec.views(init.cuda())
    emu, loss_emu = emulate_steps(init.cuda(), spec, xu8, y, B, steps, lr, adam=opt == "adam")
    tol = 1e-2 if opt == "sgd" else 0.1
    for k in ("w1", "b1", "w2", "b2"):
        r = rel(p[k] - w0[k], emu[k] - w0[k])
        assert r < tol, (k, r)
    assert abs(tr.loss_sum.item() - loss_emu) / loss_emu < 2e-3


@gpu
def test_upload_dq_slot_and_validation_count():
    """After a solo fp8 round the upload shadow (the committee's validation operand) is the
    upload blob dequantised, bit for bit, and the validation count matches the fp32 emulation of
    what the kernel computes: x_dq, the dequantised weights, fp32 biases, bf16 h."""
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
    o, P = eng.layout.offsets, eng.n_params
    up = eng.spec.views(eng.heap.view(o[f"upload_master{par}"], [P], torch.float32))
    sh = eng.spec.views(eng.heap.view(o[f"upload_shadow{par}"], [P], torch.bfloat16))
    b1, b2 = _blob_dq(eng.heap.view(eng.upq_off[par], [eng.blob_bytes], torch.uint8), eng.ql)
    assert torch.equal(sh["w1"].float(), b1) and torch.equal(sh["w2"].float(), b2[:62])
    assert torch.equal(b1, _dq_ref(up["w1"])) and torch.equal(b2[:62], _dq_ref(up["w2"]))
    x = shard.x.reshape(len(shard), -1).cuda().float() / 255.0
    assert torch.equal(eng.x_dq.float(), _dq_ref(x))
    h = torch.relu(_dq_ref(x) @ b1.t() + up["b1"]).to(torch.bfloat16).float()
    pred = (h @ b2[:62].t() + up["b2"]).argmax(-1)
    want = int((pred == shard.y.cuda()).sum())
    got = int(eng.val_correct[0].item())
    assert abs(got - want) <= 0.002 * len(shard), (got, want)
