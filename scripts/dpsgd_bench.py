"""DP-SGD cost on one GPU: a local step's forward + backward without DP-SGD, with per-example clipping
only (z = 0) and with clipping and noise, for the generic MLP (784-256-62, B 512), LoRA BERT-base and
LoRA GPT (12 layers, r 8 on q, v, B 16, S 128); and the per-example norm kernel on its own.

  python scripts/dpsgd_bench.py            -> one RESULT json line

Each variant's step is captured in one CUDA graph (the DP-SGD context is graph-capturable), replayed 5
times to warm up, then 30 times between CUDA events; the median replay is reported.  The optimizer
update is the same kernel in every variant and is left out.  The norm kernel runs at a LoRA BERT-base
site (dz [2048, 768] against u [2048, 8], 16 examples of 128 tokens), 200 launches between events;
its bytes/s counts the two bf16 operands read once.  The card's name and power limit are read in the
same process.
"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from bflc_demo_b200._native import C
from bflc_demo_b200.models.lora import LoRANet
from bflc_demo_b200.models.nets import GPT, BertBase, MLPNet
from bflc_demo_b200.ops.dpsgd import DPSGDStep

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


def workload(name):
    gen = torch.Generator().manual_seed(0)
    if name == "mlp_b512":
        net, B = MLPNet(784, 256, 62), 512
        x = net.preprocess(torch.randint(0, 256, (B, 784), generator=gen, dtype=torch.uint8).cuda())
        y = torch.randint(0, 62, (B,), generator=gen).cuda().int()
    elif name == "lora_bert_base_r8_b16_s128":
        net, B = LoRANet(BertBase(2, layers=12), 8), 16
        x = net.preprocess(torch.randint(1, 30522, (B, 128), generator=gen).cuda())
        y = torch.randint(0, 2, (B,), generator=gen).cuda().int()
    else:
        net, B = LoRANet(GPT(layers=12), 8), 16
        x = net.preprocess(torch.randint(0, 8192, (B, 128), generator=gen).cuda())
        y = torch.randint(0, 8192, (B, 128), generator=gen).cuda().int()
    master = torch.zeros(net.spec.total, device="cuda")
    net.init_(master, seed=1)
    grad = torch.zeros_like(master)
    return net, B, x, y, net.bind(master, master.to(BF), grad), grad


def main():
    out = {"card": card(), "steps_us": {}}
    word = torch.zeros(1, device="cuda", dtype=torch.int32)
    for name in ("mlp_b512", "lora_bert_base_r8_b16_s128", "lora_gpt12_r8_b16_s128"):
        net, B, x, y, bound, grad = workload(name)
        row = {}
        for variant, dp in (("off", None), ("clip", DPSGDStep(net.spec, B, 1.0, 0.0, 0, word, "cuda")),
                            ("clip_noise", DPSGDStep(net.spec, B, 1.0, 1.0, 1234, word, "cuda"))):
            def step():
                grad.zero_()
                loss = net.loss(bound, x, y)
                if dp is None:
                    loss.backward()
                else:
                    dp.begin()
                    loss.backward()
                    dp.finish(grad, 0)
            row[variant] = time_graph(step)
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
    print("RESULT " + json.dumps(out))


if __name__ == "__main__":
    main()
