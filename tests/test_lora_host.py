"""LoRA on the host: config refusals, the adapter spec's layout and the tail GEMM's compile guard."""
import os
import re
import shutil
import subprocess

import pytest
import torch

from bflc_demo_b200 import build
from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.models.lora import LoRANet, parse_targets
from bflc_demo_b200.models.nets import GPT, BertBase, MLPNet


@pytest.mark.parametrize("kw", [dict(lora_rank=4), dict(lora_rank=12), dict(lora_rank=72),
                                dict(lora_rank=8, lora_targets="q,x"), dict(lora_rank=8, lora_targets=""),
                                dict(lora_rank=8, model="mlp"), dict(lora_rank=8, dtype="fp8"),
                                dict(lora_rank=8, lora_alpha=-1.0)])
def test_config_refuses_bad_lora_settings(kw):
    base = dict(model="gpt")
    base.update(kw)
    with pytest.raises(ValueError):
        FLConfig.for_world(1, **base)


def test_config_accepts_lora_and_off_by_default():
    assert FLConfig.for_world(1, model="bert").lora_rank == 0
    c = FLConfig.for_world(1, model="bert", lora_rank=16, lora_alpha=32, lora_targets="q,k,v,o,ff1,ff2")
    assert c.lora_rank == 16


@pytest.mark.parametrize("rank,targets", [(8, "q,v"), (16, "q,k,v,o,ff1,ff2"), (64, "ff2,q")])
def test_bert_adapter_spec(rank, targets):
    net = LoRANet(BertBase(2), rank, targets=targets)
    t = parse_targets(targets)
    want = 0
    for i in range(12):
        for nm in t:
            N, K = net.base.spec.by_name[f"enc{i}.{nm}.w"].shape
            a, b = net.spec.by_name[f"enc{i}.{nm}.lora_a"], net.spec.by_name[f"enc{i}.{nm}.lora_b"]
            assert a.shape == (rank, K) and b.shape == (N, rank)
            want += rank * (N + K)
    assert net.spec.by_name["cls.w"].shape == (2, 768)
    assert sum(e.numel for e in net.spec.entries) == want + 2 * 768 + 2
    assert all(e.offset % 8 == 0 for e in net.spec.entries)         # 16-byte aligned bf16 views
    assert net.scale == 1.0


def test_bert_base_q_v_rank8_is_about_0_3m():
    assert abs(sum(e.numel for e in LoRANet(BertBase(2), 8).spec.entries) - 296_450) < 1


def test_gpt_adapter_spec_has_no_head_and_scale():
    net = LoRANet(GPT(layers=2, hidden=128, heads=2, ffn=256, vocab=512), 8, alpha=32, targets="q,ff1")
    assert "cls.w" not in net.spec.by_name and "emb.word" not in net.spec.by_name
    assert [e.name for e in net.spec.entries][:2] == ["dec0.q.lora_a", "dec0.q.lora_b"]
    assert net.spec.by_name["dec1.ff1.lora_b"].shape == (256, 8)
    assert net.scale == 4.0


def test_lora_refuses_other_models_ranks_and_base_sizes():
    with pytest.raises(ValueError):
        LoRANet(MLPNet(), 8)
    with pytest.raises(ValueError):
        LoRANet(BertBase(2, layers=1), 10)
    with pytest.raises(ValueError):
        LoRANet(BertBase(2, layers=1), 8, base_master=torch.zeros(10))


def test_bind_merges_base_and_adapters():
    base = BertBase(2, layers=1, hidden=64, heads=1, ffn=128, vocab=50, max_pos=16)
    bm = torch.arange(base.spec.total, dtype=torch.float32)
    net = LoRANet(base, 8, base_master=bm)
    master = torch.zeros(net.spec.total)
    net.init_(master, seed=1)
    grad = torch.zeros_like(master)
    b = net.bind(master, master.to(torch.bfloat16), grad)
    assert torch.equal(b.P["enc0.q.w"].flatten()[:4], bm[base.spec.offset("enc0.q.w"):][:4])
    assert b.G["enc0.q.w"] is None and b.G["emb.word"] is None and b.G["enc0.ln1.gamma"] is None
    assert b.G["cls.w"].data_ptr() == net.spec.views(grad)["cls.w"].data_ptr()
    assert set(b.lora) == {"enc0.q", "enc0.v"}
    assert torch.count_nonzero(net.spec.views(master)["enc0.q.lora_b"]) == 0
    assert torch.count_nonzero(net.spec.views(master)["enc0.q.lora_a"]) > 0


def test_base_from_checkpoint_checks_model_and_size(tmp_path):
    base = GPT(layers=1, hidden=64, heads=1, ffn=128, vocab=64, max_pos=64)
    m = torch.randn(base.spec.total)
    p = tmp_path / "ck.pt"
    torch.save(dict(config=FLConfig.for_world(1, model="gpt").to_json(), n_params=base.spec.total,
                    global_master=m), p)
    assert torch.equal(LoRANet.base_from_checkpoint(str(p), "gpt", base), m)
    with pytest.raises(ValueError):
        LoRANet.base_from_checkpoint(str(p), "bert", base)
    with pytest.raises(ValueError):
        LoRANet.base_from_checkpoint(str(p), "gpt", GPT(layers=2, hidden=64, heads=1, ffn=128, vocab=64, max_pos=64))


def test_tail_gemm_kernels_spill_free(tmp_path):
    """Both gemm_tail_kernel instantiations compile for sm_90a with zero spill bytes and no
    serialized wgmma."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("no nvcc")
    inc = [f"-I{build.CSRC / d}" for d in ("include", "ledger", "runtime")]
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, *inc, "-c", str(build.CSRC / "kernels" / "gemm_sm100.cu"),
           "-o", str(tmp_path / "g.o")]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    log = proc.stdout + proc.stderr
    assert proc.returncode == 0, log[-3000:]
    assert not [ln for ln in log.splitlines() if re.search(r"\(C75(18|20)\)", ln)]
    props = re.findall(r"Function properties for \w*?\d(gemm_tail_kernelI\w+?E)\w*\s*\n\s*"
                       r"\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert {n for n, _, _ in props} == {"gemm_tail_kernelILi64E", "gemm_tail_kernelILi128E"}, props
    for name, st, ld in props:
        assert st == "0" and ld == "0", f"{name}: {st} B spill stores / {ld} B spill loads"


# ------------------------------------------------------------------ fp64 LoRA reference
def lora_linear64(x, w, b, A, B, scale, round_u=None):
    """fp64 LoRA linear ``x W^T + b + scale (x A^T) B^T`` (pre-activation); ``round_u`` an optional
    hook on u = scale x A^T (the GPU suites' bf16 emulation rounds it where the kernels store it)."""
    u = scale * (x @ A.T)
    if round_u is not None:
        u = round_u(u)
    z = x @ w.T + u @ B.T
    return z if b is None else z + b


@pytest.mark.parametrize("r,scale", [(8, 1.0), (16, 2.0), (64, 0.25)])
def test_fp64_lora_linear_matches_stock_torch_modules(r, scale):
    """The reference against torch.nn.Linear for W, b plus two bias-free nn.Linear adapters, values
    and autograd gradients, and against the merged weight W + s B A."""
    torch.manual_seed(r)
    M, N, K = 12, 40, 24
    base = torch.nn.Linear(K, N).double()
    down, up = torch.nn.Linear(K, r, bias=False).double(), torch.nn.Linear(r, N, bias=False).double()
    x = torch.randn(M, K, dtype=torch.float64, requires_grad=True)
    y_stock = base(x) + scale * up(down(x))
    A = down.weight.detach().clone().requires_grad_(True)
    B = up.weight.detach().clone().requires_grad_(True)
    x2 = x.detach().clone().requires_grad_(True)
    y_ref = lora_linear64(x2, base.weight.detach(), base.bias.detach(), A, B, scale)
    assert torch.allclose(y_ref, y_stock, rtol=1e-12, atol=1e-12)
    merged = x.detach() @ (base.weight.detach() + scale * B.detach() @ A.detach()).T + base.bias.detach()
    assert torch.allclose(y_ref.detach(), merged, rtol=1e-12, atol=1e-12)
    dy = torch.randn(M, N, dtype=torch.float64)
    y_stock.backward(dy)
    y_ref.backward(dy)
    assert torch.allclose(A.grad, down.weight.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(B.grad, up.weight.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(x2.grad, x.grad, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------ command line
@pytest.mark.parametrize("argv", [
    ["--model", "mlp", "--lora-rank", "8"],
    ["--model", "lenet5", "--lora-rank", "8"],
    ["--model", "resnet18", "--lora-rank", "8"],
    ["--model", "mlp", "--generic", "--lora-rank", "8"],
    ["--model", "gpt", "--lora-rank", "12"],
    ["--model", "gpt", "--lora-rank", "128"],
    ["--model", "bert", "--lora-rank", "8", "--lora-targets", "q,qq"],
    ["--model", "bert", "--lora-rank", "8", "--dtype", "fp8"],
    ["--model", "gpt", "--lora-rank", "8", "--lora-alpha", "-2"],
    ["--model", "gpt", "--lora-targets", "q,k"],
    ["--model", "gpt", "--lora-base", "base.pt"],
    ["--model", "gpt", "--lora-rank", "8", "--lora-base", "/nonexistent/base.pt"],
])
def test_run_rejects_lora_flag_combinations(argv):
    from bflc_demo_b200 import run
    with pytest.raises(SystemExit) as e:
        run.main(argv + ["--rounds", "1"])
    assert e.value.code == 2


def test_fused_engine_refuses_lora():
    from bflc_demo_b200.engine.fused import FusedEngine
    cfg = FLConfig.for_world(1, model="mlp")
    cfg.lora_rank = 8
    with pytest.raises(ValueError, match="LoRA"):
        FusedEngine(cfg, None)


def test_config_and_net_must_agree_on_lora():
    from bflc_demo_b200.models.lora import check_net_matches_config, lora_net_from_config
    base = GPT(layers=1, hidden=64, heads=1, ffn=128, vocab=64)
    on = FLConfig.for_world(1, model="gpt", lora_rank=8, lora_alpha=16, lora_targets="q,ff1")
    off = FLConfig.for_world(1, model="gpt")
    net = lora_net_from_config(on, base)
    assert (net.rank, net.scale, net.targets) == (8, 2.0, ("q", "ff1"))
    check_net_matches_config(on, net)
    check_net_matches_config(off, base)
    with pytest.raises(ValueError):
        check_net_matches_config(on, base)            # lora_rank set, plain net: would train every weight
    with pytest.raises(ValueError):
        check_net_matches_config(off, net)            # a LoRANet under a config that says LoRA is off
    for other in (dict(lora_rank=16), dict(lora_alpha=8), dict(lora_targets="q,v")):
        kw = dict(model="gpt", lora_rank=8, lora_alpha=16, lora_targets="q,ff1")
        kw.update(other)
        with pytest.raises(ValueError):
            check_net_matches_config(FLConfig.for_world(1, **kw), net)


def test_base_checkpoint_shape_lora_run_and_rank_files(tmp_path):
    import json
    from bflc_demo_b200.models.lora import model_shape
    a = GPT(layers=2, hidden=64, heads=1, ffn=128, vocab=64, max_pos=64)
    b = GPT(layers=2, hidden=64, heads=1, ffn=128, vocab=64, max_pos=64)
    b.Hd = 65                                          # same count, another recorded shape
    m = torch.randn(a.spec.total)
    blob = dict(config=FLConfig.for_world(1, model="gpt").to_json(), n_params=a.spec.total, global_master=m,
                model_shape=json.dumps(model_shape(a)))
    torch.save(blob, tmp_path / "ck.pt.rank0")         # a multi-rank run's files
    assert torch.equal(LoRANet.base_from_checkpoint(str(tmp_path / "ck.pt"), "gpt", a), m)
    with pytest.raises(ValueError, match="shape"):
        LoRANet.base_from_checkpoint(str(tmp_path / "ck.pt"), "gpt", b)
    blob["config"] = FLConfig.for_world(1, model="gpt", lora_rank=8).to_json()
    torch.save(blob, tmp_path / "lora.pt")
    with pytest.raises(ValueError, match="LoRA run"):
        LoRANet.base_from_checkpoint(str(tmp_path / "lora.pt"), "gpt", a)
