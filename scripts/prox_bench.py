"""Cost and effect of FedProx local training (prox_mu > 0), one JSON line per measurement.

  python scripts/prox_bench.py trainer     # persistent trainer: us per local step from the device stamps,
                                           # mu = 0 vs mu > 0, bf16 / fp8 x SGD / Adam (B 512, 8 steps)
  python scripts/prox_bench.py optim       # recipe k_optim at BERT-base size (110M fp32), with and without
                                           # the anchor: time and GB/s of the bytes it must move
  python scripts/prox_bench.py effect      # solo FusedEngine, Dirichlet(0.1) shards, 30 rounds, mu in
                                           # {0, 0.01, 0.1}: test accuracy per round, final ||upload - global||

Every line names the card and its power limit."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from bflc_demo_b200._native import C  # noqa: E402
from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec, sf_bytes  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        q = torch.cuda.get_device_name()
    return q


def trainer():
    B, steps, reps = 512, 8, 30
    spec = mlp_spec(784, 256, 62)
    init = torch.empty(spec.total)
    spec.init_(init, seed=2)
    U = (torch.rand(B * steps, 784, device="cuda") * 255).to(torch.uint8)
    X = torch.empty(B * steps, 784, device="cuda", dtype=torch.bfloat16)
    XQ = torch.zeros(B * steps, 784, device="cuda", dtype=torch.uint8)
    XSF = torch.full((sf_bytes(B * steps, 784),), 127, device="cuda", dtype=torch.uint8)
    XDQ = torch.empty(B * steps, 784, device="cuda", dtype=torch.bfloat16)
    C().prep_inputs(U, X, XQ, XSF, 1.0 / 255.0, XDQ)
    Y = torch.randint(0, 62, (B * steps,), device="cuda", dtype=torch.int32)
    anchor = init.cuda() + 0.01
    for fp8 in (False, True):
        for adam in (False, True):
            res = {}
            for mu in (0.0, 0.01):
                master = init.cuda().clone()
                tr = FlatMLP(spec, master, master.bfloat16(), torch.zeros_like(master), B,
                             lr=1e-3 if adam else 0.05, optimizer="adam" if adam else "sgd", fp8=fp8,
                             prox_mu=mu, anchor=anchor if mu > 0 else None)
                if fp8:
                    tr.quantize_weights()
                bar = torch.zeros(1, device="cuda", dtype=torch.int32)
                dbg = torch.zeros(steps, 32, device="cuda", dtype=torch.int64)
                per = []
                for it in range(reps + 3):
                    bar.zero_()
                    dbg.zero_()
                    tr.train_epoch_fused(X, Y, steps, bar.data_ptr(), dbg, x_dq=XDQ if fp8 else None)
                    torch.cuda.synchronize()
                    d = dbg.cpu().double()
                    if it >= 3:      # step s ends where step s + 1 begins; the last step ends at slot 4
                        per.append(float(d[steps - 1, 4] - d[0, 0]) / 1e3 / steps)
                per.sort()
                res[mu] = per[len(per) // 2]
            print(json.dumps(dict(bench="prox_trainer", dtype="fp8" if fp8 else "bf16", opt="adam" if adam else "sgd",
                                  us_per_step_mu0=round(res[0.0], 3), us_per_step_prox=round(res[0.01], 3),
                                  delta_us=round(res[0.01] - res[0.0], 3), card=card())), flush=True)


def optim():
    n = 110_000_000          # BERT-base parameter count
    master = torch.randn(n, device="cuda")
    grad = torch.randn(n, device="cuda") * 1e-3
    shadow = master.bfloat16()
    m, v = torch.zeros_like(master), torch.zeros_like(master)
    anchor = master + 0.01
    for adam in (False, True):
        for prox in (False, True):
            kw = dict(anchor=anchor, prox_mu=0.01) if prox else {}
            args = (adam, master, grad, shadow, m if adam else None, v if adam else None, 1e-4, 0.9, 0.999, 1e-8,
                    1, 0, 0.0, None, 0, 0, 0, None)
            for _ in range(5):
                C().optim_recipe_step(*args, zero_grad=False, **kw)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 50
            e0.record()
            for _ in range(reps):
                C().optim_recipe_step(*args, zero_grad=False, **kw)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            # bytes per parameter: w read + write, g read, bf16 shadow write (+ m, v read + write, + anchor read)
            bpp = 4 + 4 + 4 + 2 + (16 if adam else 0) + (4 if prox else 0)
            print(json.dumps(dict(bench="prox_optim", opt="adam" if adam else "sgd", anchor=prox, n=n,
                                  ms=round(ms, 4), bytes_per_param=bpp, GBps=round(n * bpp / ms / 1e6, 1),
                                  card=card())), flush=True)


def effect():
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    rounds = 30
    for mu in (0.0, 0.01, 0.1):
        cfg = FLConfig.for_world(1, model="mlp", batch_size=512, samples_per_client=4096, learning_rate=0.05,
                                 ring_slots=1024, prox_mu=mu, non_iid_alpha=0.1, seed=1)
        shard = femnist_like(1, 4096, seed=7, only=0, alpha=0.1)[0]
        test = femnist_like(1, 2048, seed=7, only=0)[0]
        eng = FusedEngine(cfg, shard)
        eng.capture()
        accs = [round(eng.evaluate(test), 4)]
        for _ in range(rounds - 1):
            g0 = eng.global_master.clone()
            eng.run_round()
            accs.append(round(eng.evaluate(test), 4))
        torch.cuda.synchronize()
        o, P = eng.layout.offsets, eng.n_params
        ep = eng.read_state()["epoch"]
        up = eng.heap.view(o[f"upload_master{(ep - 1) & 1}"], [P], torch.float32)
        dist = float((up - g0).norm())
        print(json.dumps(dict(bench="prox_effect", prox_mu=mu, non_iid_alpha=0.1, rounds=rounds, test_acc=accs,
                              final_upload_minus_global=round(dist, 6), mismatches=len(eng.drain_blocks()),
                              card=card())), flush=True)
        del eng


if __name__ == "__main__":
    what = sys.argv[1:] or ["trainer", "optim", "effect"]
    for w in what:
        {"trainer": trainer, "optim": optim, "effect": effect}[w]()
