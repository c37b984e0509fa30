"""DP-SGD cost on one GPU: a local step's forward + backward without DP-SGD, with per-example clipping
only (z = 0) and with clipping and noise, for the generic MLP (784-256-62, B 512), LoRA BERT-base and
LoRA GPT (12 layers, r 8 on q, v, B 16, S 128), full BERT-base and full GPT (12 layers, every parameter
clipped: ``dpsgd_full_model``) at B 16 with S 128 and S 512, LeNet-5 (B 128) and the GroupNorm ResNet-18
(B 64, 32 x 32; ``dpsgd_conv``); and the per-example norm kernels on their own.

  python scripts/dpsgd_bench.py            -> one RESULT json line

Each variant's step is captured in one CUDA graph (the DP-SGD context is graph-capturable), replayed 5
times to warm up, then 30 times between CUDA events; the median replay is reported.  The optimizer
update is the same kernel in every variant and is left out.  The norm kernel runs at a LoRA BERT-base
site (dz [2048, 768] against u [2048, 8], 16 examples of 128 tokens), 200 launches between events;
its bytes/s counts the two bf16 operands read once.  The Gram-form kernel runs at a BERT-base ff1 site
(dz [2048, 3072] against x [2048, 768] with its bias, 16 examples of 128 tokens), 50 launches between
events; its FLOP/s counts 2 R^2 (a + b) B, the two Grams' multiply-adds over every tile pair's full
64 x 64 square (the pairs i < j stand for their mirror images, so this is the work the sum needs).  The
convolution sites run at B 64: a ResNet stage-1 3x3 64->64 site (R 1024, patches 576 wide) by im2col plus
product tiles and by the implicit weight-gradient GEMM's per-example mode, and a stage-4 3x3 512->512 site (R 16, patches 4608 wide) by product tiles and by the Gram
form, 20 launches between events each.  The convolutional models' DP-SGD variants run with deterministic
convolutions, as GenericFedEngine runs them.  The card's name and power limit are read in the same process.

Poisson sampling (``dpsgd_sampling = "poisson"``, ``poisson`` in the RESULT): the sampler's one launch per round at
(S, steps) = (4096, 8) and (60000, 117) with B 512, 50 launches between events; and one clipped and noised local
step at the capacity (the slots a Poisson step computes on, padding included) against the partition step at B, for
the MLP (B 512 of S 4096: cap 672) and LoRA BERT-base (B 16 of S 2048: cap 56), graph-replayed as above.

  python scripts/dpsgd_bench.py --poisson  -> only the Poisson figures

DP-SGD in the persistent MLP trainer (``dpsgd_fused``, ``fused`` in the RESULT): the trainer's local step from
its %globaltimer stamps (CTA 0, as scripts/mlp_phases.py reads them) without and with DP-SGD (C 1, z 1), bf16
and fp8, B 512, Adam, one 8-step launch per sample with the cold first step skipped, alternated three times:
the whole step, the part up to the barrier after the fused chain (fwd1, softmax, dh and, with DP-SGD, the norm
exchange, the clip factors and the dlogits / db2 stores that wait for them) and phase B.  Then FusedEngine
rounds/s at bench.py's default config (B 512 of S 4096, Adam, fp8) without and with DP-SGD, alternated three
times (20 replayed rounds between CUDA events), beside the generic MLP's DP-SGD step at B 512.

  python scripts/dpsgd_bench.py --fused    -> only the persistent-trainer figures

DP-SGD on packed variable-length BERT (``dpsgd_packed``, ``packed`` in the RESULT): LoRA BERT-base (r 8 on q, v) and
full BERT-base at B 16, S 512, with lengths from ``tokens_like(min_len=32, seq_len=512)`` at a fixed seed, four
graph-replayed steps each: padded and packed, without DP-SGD and with clipping and noise (C 1, z 1).  Beside them
the counts the lengths give: token rows (B S padded, T packed) and the Gram-form FLOPs of the full model's sites,
2 L^2 (a + b) per example and site (the embeddings' one-hot side costs nothing).  Then the Gram kernel at a BERT-base
ff1 site over the same lengths, packed (k_packed_gram) against padded to 512 rows (k_pe_gram), 20 launches between
events each.  The packed model runs only where a sample's tokens are, so the counts say what packing can save;
the timings say what it does.

  python scripts/dpsgd_bench.py --packed   -> only the packed-BERT figures
"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from bflc_demo_b200._native import C
from bflc_demo_b200.models.lora import LoRANet
from bflc_demo_b200.models.nets import GPT, BertBase, LeNet5, MLPNet, ResNet18
from bflc_demo_b200.ops import nn as F
from bflc_demo_b200.ops.dpsgd import DPSGDStep, PoissonSampler

BF = torch.bfloat16


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return {"name": name, "nvidia_smi": q}
    except (OSError, subprocess.SubprocessError):
        return {"name": name, "nvidia_smi": "not available"}


def time_graph(step):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    for _ in range(5):
        g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(30):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return round(ts[len(ts) // 2], 1)


def workload(name, rows=None):
    """(net, B, x, y, bound, grad) of a named step; ``rows`` (default B): the examples x and y hold."""
    gen = torch.Generator().manual_seed(0)
    if name == "mlp_b512":
        net, B = MLPNet(784, 256, 62), 512
        x = net.preprocess(torch.randint(0, 256, (B, 784), generator=gen, dtype=torch.uint8).cuda())
        y = torch.randint(0, 62, (B,), generator=gen).cuda().int()
    elif name == "lora_bert_base_r8_b16_s128":
        net, B = LoRANet(BertBase(2, layers=12), 8), 16
        x = net.preprocess(torch.randint(1, 30522, (B, 128), generator=gen).cuda())
        y = torch.randint(0, 2, (B,), generator=gen).cuda().int()
    elif name in ("lenet5_b128", "resnet18_gn_b64"):
        net, B = (LeNet5(), 128) if name == "lenet5_b128" else (ResNet18(norm="group"), 64)
        x = net.preprocess(torch.randint(0, 256, (B, 3, 32, 32), generator=gen, dtype=torch.uint8).cuda())
        y = torch.randint(0, 10, (B,), generator=gen).cuda().int()
    elif name.startswith("full_bert_base"):
        S = int(name.rsplit("_s", 1)[1])
        net, B = BertBase(2, layers=12), 16
        x = net.preprocess(torch.randint(1, 30522, (B, S), generator=gen).cuda())
        y = torch.randint(0, 2, (B,), generator=gen).cuda().int()
    else:
        S = int(name.rsplit("_s", 1)[1])
        net, B = (GPT(layers=12) if name.startswith("full") else LoRANet(GPT(layers=12), 8)), 16
        x = net.preprocess(torch.randint(0, 8192, (B, S), generator=gen).cuda())
        y = torch.randint(0, 8192, (B, S), generator=gen).cuda().int()
    if rows is not None:      # more rows of the same kind, cycling through the B drawn above
        pick = torch.arange(rows, device="cuda") % B
        x, y = x.index_select(0, pick), y.index_select(0, pick)
    master = torch.zeros(net.spec.total, device="cuda")
    net.init_(master, seed=1)
    grad = torch.zeros_like(master)
    return net, B, x, y, net.bind(master, master.to(BF), grad), grad


def poisson():
    word = torch.zeros(1, device="cuda", dtype=torch.int32)
    res = {"sampler_us": {}, "steps_us": {}}
    for S, steps in ((4096, 8), (60000, 117)):
        ps = PoissonSampler(S, 512, steps, 0x5EED, "cuda")
        res["sampler_us"][f"S{S}_steps{steps}_B512_cap{ps.cap}"] = _events(lambda: ps.sample(word), 50)
    for name, S in (("mlp_b512", 4096), ("lora_bert_base_r8_b16_s128", 2048)):
        _, B, *_ = workload(name)
        cap = PoissonSampler(S, B, 1, 1, "cuda").cap
        row = {"B": B, "cap": cap}
        for variant, rows in (("partition", B), ("poisson", cap)):
            net, _, x, y, bound, grad = workload(name, rows)
            dp = DPSGDStep(net.spec, rows, 1.0, 1.0, 1234, word, "cuda", norm_batch=B)
            n_valid = torch.full((1,), B, device="cuda", dtype=torch.int32) if rows != B else None

            def step():
                grad.zero_()
                loss = net.loss(bound, x, y)
                dp.begin()
                (loss * (rows / B) if rows != B else loss).backward()
                dp.finish(grad, 0, n_valid=n_valid)
            prev = F.set_deterministic(True)
            row[f"{variant}_us"] = time_graph(step)
            F.set_deterministic(prev)
            del net, bound, grad
            torch.cuda.empty_cache()
        row["ratio"] = round(row["poisson_us"] / row["partition_us"], 3)
        res["steps_us"][name] = row
    return res


def fused():
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec
    B, steps = 512, 8
    spec = mlp_spec(784, 256, 62)
    init = torch.empty(spec.total)
    spec.init_(init, seed=2)
    U = (torch.rand(B * steps, 784, device="cuda") * 255).to(torch.uint8)
    X = torch.empty(B * steps, 784, device="cuda", dtype=BF)
    XDQ = torch.empty_like(X)
    C().prep_inputs(U, X, None, None, 1.0 / 255.0, XDQ)
    Y = torch.randint(0, 62, (B * steps,), device="cuda", dtype=torch.int32)
    word = torch.zeros(1, device="cuda", dtype=torch.int32)
    res = {"trainer_us": {}, "engine_rounds_per_s": {}}
    for fp8 in (False, True):
        trs = {}
        for name, dp in (("off", {}), ("dpsgd", dict(dpsgd_clip=1.0, dpsgd_noise=1.0, dpsgd_seed=1234))):
            m = init.cuda().clone()
            trs[name] = FlatMLP(spec, m, m.bfloat16(), torch.zeros_like(m), B, optimizer="adam", lr=1e-3,
                                step_dev_ptr=word.data_ptr(), fp8=fp8, **dp)
            if fp8:
                trs[name].quantize_weights()
        bar = torch.zeros(1, device="cuda", dtype=torch.int32)
        dbg = torch.zeros(steps, 32, device="cuda", dtype=torch.int64)
        rows = {k: {"step": [], "to_chain_barrier": [], "phase_B": []} for k in trs}
        for rep in range(4):
            for k, tr in trs.items():
                bar.zero_()
                dbg.zero_()
                tr.train_epoch_fused(X, Y, steps, bar.data_ptr(), dbg, x_dq=XDQ if fp8 else None)
                torch.cuda.synchronize()
                if rep == 0:      # warm-up
                    continue
                d = dbg.cpu().double()
                for key, a, b in (("step", 0, 4), ("to_chain_barrier", 0, 2), ("phase_B", 2, 4)):
                    rows[k][key].append(round(float((d[1:, b] - d[1:, a]).mean()) / 1e3, 2))
        res["trainer_us"]["fp8" if fp8 else "bf16"] = rows
    engs = {}
    for name, dp in (("off", {}), ("dpsgd", dict(dpsgd_clip=1.0, dpsgd_noise=1.0, dpsgd_fused=True))):
        cfg = FLConfig.for_world(1, model="mlp", batch_size=B, samples_per_client=4096, learning_rate=1e-3,
                                 optimizer="adam", dtype="fp8", **dp)
        engs[name] = FusedEngine(cfg, femnist_like(1, 4096, seed=7, only=0)[0])
        engs[name].capture()
    for rep in range(3):
        for k, e in engs.items():
            for _ in range(3):
                e.run_round()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(e.stream)
            for _ in range(20):
                e.run_round()
            e1.record(e.stream)
            e1.synchronize()
            res["engine_rounds_per_s"].setdefault(k, []).append(round(20 / (e0.elapsed_time(e1) * 1e-3), 1))
    for e in engs.values():
        assert e.drain_blocks() == []
    net, Bm, x, y, bound, grad = workload("mlp_b512")
    dp = DPSGDStep(net.spec, Bm, 1.0, 1.0, 1234, word, "cuda")

    def step():
        grad.zero_()
        loss = net.loss(bound, x, y)
        dp.begin()
        loss.backward()
        dp.finish(grad, 0)
    prev = F.set_deterministic(True)
    res["generic_mlp_b512_clip_noise_step_us"] = time_graph(step)
    F.set_deterministic(prev)
    return res


def packed():
    from bflc_demo_b200.data.synthetic import tokens_like
    B, S, H, FF, L = 16, 512, 768, 3072, 12
    ids = tokens_like(1, B, seed=5, seq_len=S, min_len=32)[0].x.cuda()
    lens = (ids != 0).sum(1).tolist()
    T = sum(lens)
    # Gram sites of full BERT-base: per layer q, k, v, o (768 x 768 + bias), ff1 (3072 x 768 + bias), ff2
    # (768 x 3072 + bias); the word and position embeddings (one-hot side exact: 768 only)
    widths = [2 * H + 1] * 4 * L + [FF + H + 1] * L + [H + FF + 1] * L + [H] * 2
    gram = {"padded": sum(2 * S * S * w * B for w in widths), "packed": sum(2 * n * n * w for w in widths for n in lens)}
    res = {"lengths": lens, "token_rows": {"padded": B * S, "packed": T},
           "full_model_gram_GFLOP": {k: round(v / 1e9, 1) for k, v in gram.items()},
           "gram_ratio": round(gram["padded"] / gram["packed"], 2), "rows_ratio": round(B * S / T, 2),
           "steps_us": {}}
    word = torch.zeros(1, device="cuda", dtype=torch.int32)
    y = torch.randint(0, 2, (B,), generator=torch.Generator().manual_seed(5)).cuda().int()
    for name in ("lora_bert_base_r8_b16_s512", "full_bert_base_b16_s512"):
        row = {}
        for layout in ("padded", "packed"):
            base = BertBase(2, layers=L, pad_id=0, packed=layout == "packed")
            net = LoRANet(base, 8) if name.startswith("lora") else base
            x = net.preprocess(ids)
            master = torch.zeros(net.spec.total, device="cuda")
            net.init_(master, seed=1)
            grad = torch.zeros_like(master)
            bound = net.bind(master, master.to(BF), grad)
            seg = x if layout == "packed" else None
            for variant, dp in (("off", None), ("clip_noise", DPSGDStep(net.spec, B, 1.0, 1.0, 1234, word, "cuda"))):
                def step():
                    grad.zero_()
                    loss = net.loss(bound, x, y)
                    if dp is None:
                        loss.backward()
                    else:
                        dp.begin(seg)
                        loss.backward()
                        dp.finish(grad, 0)
                prev = F.set_deterministic(dp is not None)
                row[f"{layout}_{variant}"] = time_graph(step)
                F.set_deterministic(prev)
            del net, base, bound, grad, master
            torch.cuda.empty_cache()
        row["dp_packed_speedup"] = round(row["padded_clip_noise"] / row["packed_clip_noise"], 2)
        res["steps_us"][name] = row
    gen = torch.Generator(device="cuda").manual_seed(6)
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), device="cuda", dtype=torch.int32)
    site = {}
    for layout, rows in (("padded", B * S), ("packed", T)):
        x = torch.randn(rows, H, generator=gen, device="cuda").to(BF)
        dz = torch.randn(rows, FF, generator=gen, device="cuda").to(BF)
        part = torch.empty(C().dpsgd_gram_pairs(S, True) * B, device="cuda")
        kw = {"cu_seqlens": cu} if layout == "packed" else {}
        site[f"{layout}_us"] = _events(lambda: C().dpsgd_pe_gram(x, x, S, 1.0, part, p1=dz, p2=dz, mode=0, **kw), 20)
    site["shape"] = f"ff1: dz [rows, 3072], x [rows, 768] + bias, B 16, max_len 512; rows {B * S} padded, {T} packed"
    res["ff1_gram"] = site
    return res


def main():
    if "--packed" in sys.argv[1:]:
        print("RESULT " + json.dumps({"card": card(), "packed": packed()}))
        return
    if "--fused" in sys.argv[1:]:
        print("RESULT " + json.dumps({"card": card(), "fused": fused()}))
        return
    if "--poisson" in sys.argv[1:]:
        print("RESULT " + json.dumps({"card": card(), "poisson": poisson()}))
        return
    out = {"card": card(), "steps_us": {}}
    word = torch.zeros(1, device="cuda", dtype=torch.int32)
    for name in ("mlp_b512", "lora_bert_base_r8_b16_s128", "lora_gpt12_r8_b16_s128", "full_bert_base_b16_s128",
                 "full_gpt12_b16_s128", "full_bert_base_b16_s512", "full_gpt12_b16_s512", "lenet5_b128",
                 "resnet18_gn_b64"):
        net, B, x, y, bound, grad = workload(name)
        row = {}
        conv = name in ("lenet5_b128", "resnet18_gn_b64")
        for variant, dp in (("off", None), ("clip", DPSGDStep(net.spec, B, 1.0, 0.0, 0, word, "cuda", conv=conv)),
                            ("clip_noise", DPSGDStep(net.spec, B, 1.0, 1.0, 1234, word, "cuda", conv=conv))):
            def step():
                grad.zero_()
                loss = net.loss(bound, x, y)
                if dp is None:
                    loss.backward()
                else:
                    dp.begin()
                    loss.backward()
                    dp.finish(grad, 0)
            prev = F.set_deterministic(dp is not None)
            row[variant] = time_graph(step)
            F.set_deterministic(prev)
        row["params"] = net.spec.total
        out["steps_us"][name] = row
        del net, bound, grad
        torch.cuda.empty_cache()
    gen = torch.Generator(device="cuda").manual_seed(2)
    dz = torch.randn(2048, 768, generator=gen, device="cuda").to(BF)
    u = torch.randn(2048, 8, generator=gen, device="cuda").to(BF)
    part = torch.empty(12 * 16, device="cuda")
    for _ in range(20):
        C().dpsgd_pe_norm(dz, u, 128, part)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(200):
        C().dpsgd_pe_norm(dz, u, 128, part)
    e1.record()
    e1.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / 200
    nbytes = (dz.numel() + u.numel()) * 2
    out["pe_norm"] = {"shape": "dz 2048x768, u 2048x8, R 128", "us": round(us, 2),
                      "GB_per_s": round(nbytes / (us * 1e-6) / 1e9, 1)}
    x = torch.randn(2048, 768, generator=gen, device="cuda").to(BF)
    dz = torch.randn(2048, 3072, generator=gen, device="cuda").to(BF)
    R, B = 128, 16
    part = torch.empty(C().dpsgd_gram_pairs(R, True) * B, device="cuda")
    for _ in range(10):
        C().dpsgd_pe_gram(x, x, R, 1.0, part, p1=dz, p2=dz, mode=0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        C().dpsgd_pe_gram(x, x, R, 1.0, part, p1=dz, p2=dz, mode=0)
    e1.record()
    e1.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / 50
    flops = 2 * R * R * (3072 + 768) * B
    out["pe_gram"] = {"shape": "ff1: dz 2048x3072, x 2048x768 + bias, R 128, B 16", "us": round(us, 2),
                      "TFLOP_per_s": round(flops / (us * 1e-6) / 1e12, 1)}
    out["conv_sites"] = conv_sites()
    out["poisson"] = poisson()
    out["fused"] = fused()
    print("RESULT " + json.dumps(out))


def _events(fn, n):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return round(e0.elapsed_time(e1) * 1e3 / n, 2)


def conv_sites():
    gen = torch.Generator(device="cuda").manual_seed(3)
    B, res = 64, {}
    # stage 1: x [64, 32, 32, 64], 3x3 pad 1 -> R 1024, patches 576 wide
    x = torch.randn(B, 32, 32, 64, generator=gen, device="cuda").to(BF)
    dz = torch.randn(B * 1024, 64, generator=gen, device="cuda").to(BF)
    col = torch.empty(B * 1024, 576, device="cuda", dtype=BF)
    part = torch.empty(C().dpsgd_norm_tiles(64, 576, False) * B, device="cuda")

    def stage1():
        C().im2col(x, col, B, 64, 32, 32, 3, 3, 1, 1, 32, 32)
        C().dpsgd_pe_norm(dz, col, 1024, part)
    gemm_part = torch.empty(C().conv_dw_norm_tiles(64, 576) * B, device="cuda")
    res["stage1_64x576_R1024"] = {
        "im2col_plus_tiles_us": _events(stage1, 20),
        "tiles_us": _events(lambda: C().dpsgd_pe_norm(dz, col, 1024, part), 20),
        "implicit_gemm_norm_us": _events(lambda: C().conv_dw_groups(x, dz, gemm_part, B, 32, 32, 64, 32, 32, 3, 3,
                                                                    1, 1, B, True), 20)}
    # stage 4: x [64, 4, 4, 512] -> R 16, patches 4608 wide
    dz = torch.randn(B * 16, 512, generator=gen, device="cuda").to(BF)
    col = torch.randn(B * 16, 4608, generator=gen, device="cuda").to(BF)
    tiles = torch.empty(C().dpsgd_norm_tiles(512, 4608, False) * B, device="cuda")
    pairs = torch.empty(C().dpsgd_gram_pairs(16, True) * B, device="cuda")
    res["stage4_512x4608_R16"] = {
        "tiles_us": _events(lambda: C().dpsgd_pe_norm(dz, col, 16, tiles), 20),
        "gram_us": _events(lambda: C().dpsgd_pe_gram(col, col, 16, 0.0, pairs, p1=dz, p2=dz, mode=0), 20)}
    return res


if __name__ == "__main__":
    main()
