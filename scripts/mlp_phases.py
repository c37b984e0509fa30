"""In-kernel %globaltimer phase stamps of the persistent trainer (CTA 0), one variant per process:
BFLC_MLP_CHAIN / BFLC_MLP_EPIOPT select the phase plan, --fp8 the block-scaled fp8 forward,
--adam the optimizer.  Prints mean per-slot deltas (us)."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from bflc_demo_b200._native import C
from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec, sf_bytes

def main():
    B, steps = 512, 8
    fp8, adam = "--fp8" in sys.argv, "--adam" in sys.argv
    spec = mlp_spec(784, 256, 62)
    init = torch.empty(spec.total); spec.init_(init, seed=2)
    master = init.cuda().clone(); shadow = master.bfloat16(); grad = torch.zeros_like(master)
    U = (torch.rand(B * steps, 784, device="cuda") * 255).to(torch.uint8)
    X = torch.empty(B * steps, 784, device="cuda", dtype=torch.bfloat16)
    XQ = torch.zeros(B * steps, 784, device="cuda", dtype=torch.uint8)
    XSF = torch.full((sf_bytes(B * steps, 784),), 127, device="cuda", dtype=torch.uint8)
    C().prep_inputs(U, X, XQ, XSF, 1.0 / 255.0)
    Y = torch.randint(0, 62, (B * steps,), device="cuda", dtype=torch.int32)
    tr = FlatMLP(spec, master, shadow, grad, B, lr=1e-3 if adam else 0.05, optimizer="adam" if adam else "sgd",
                 fp8=fp8)
    if fp8:
        tr.quantize_weights()
    bar = torch.zeros(1, device="cuda", dtype=torch.int32)
    dbg = torch.zeros(steps, 32, device="cuda", dtype=torch.int64)
    tot = []
    for it in range(6):
        bar.zero_(); dbg.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        tr.train_epoch_fused(X, Y, steps, bar.data_ptr(), dbg, x_q=XQ, x_sf=XSF)
        e1.record(); torch.cuda.synchronize()
        tot.append(e0.elapsed_time(e1) * 1e3)
    d = dbg.cpu().double()
    chain = os.environ.get("BFLC_MLP_CHAIN", "4")
    names = {0: "step_begin", 1: "after_P1_barrier", 6: "chain:h/acc_h ready", 7: "chain:E1 done",
             8: "chain:logits ready", 12: "chain:E2 max pass done", 13: "chain:E2 tile written",
             14: "chain:E2 arrived", 9: "chain:E2 done", 10: "chain:dh acc ready", 11: "chain:E3 done",
             2: "after_chain/P3_barrier", 3: "B tile done", 4: "after_B_barrier", 5: "after_P5_barrier",
             16: "P1:acc ready", 17: "P1:epilogue done", 18: "B:acc ready", 19: "B:epilogue done"}
    order = [0, 16, 17, 1, 6, 7, 8, 12, 13, 14, 9, 10, 11, 2, 18, 19, 3, 4, 5]
    if chain == "4":   # no barrier after P1: the fwd1 epilogue hands h over inside the cluster
        names.update({1: "P1:h slice handed to the cluster", 6: "chain:h tile complete"})
        order = [0, 16, 1, 17, 6, 7, 8, 12, 13, 14, 9, 10, 11, 2, 18, 19, 3, 4, 5]
    rows = {}
    for s in range(1, steps):          # skip the cold first step
        t0 = d[s, 0].item()
        for k in order:
            if d[s, k].item() > 0:
                rows.setdefault(names[k], []).append((d[s, k].item() - t0) / 1e3)
    nxt = [(d[s + 1, 0] - d[s, 0]).item() / 1e3 for s in range(1, steps - 1)]
    out = {"fp8": fp8, "adam": adam,
           "chain": chain, "epiopt": os.environ.get("BFLC_MLP_EPIOPT", "1"),
           "kernel_us_min": min(tot), "step_us_mean": sum(nxt) / len(nxt),
           "since_step_begin_us": {k: round(sum(v) / len(v), 2) for k, v in rows.items()}}
    print("PHASES " + json.dumps(out))

if __name__ == "__main__":
    main()
