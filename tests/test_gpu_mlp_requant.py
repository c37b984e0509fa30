"""MXFP8 re-quantisation in the persistent trainer's optimizer epilogue (E_OPT, fp8 mode): after
every step the epilogue rewrites the weights' MXFP8 work blob (e4m3 bytes + UE8M0 scale chunks) and
their exactly dequantised bf16 copy work_dq from the updated fp32 master.  Both must be bit-identical
to what the stand-alone quantiser (quantize_mlp_blob) makes of the same master, for every phase plan
that runs the epilogue, both optimizers and batch sizes whose last weight tile has a partial K-group
(in_dim 784 = 24.5 groups of 32)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("plan,opt,B,steps", [(4, "adam", 512, 1), (4, "adam", 512, 3), (4, "sgd", 256, 2),
                                              (4, "sgd", 128, 1), (3, "adam", 256, 2), (3, "sgd", 512, 1)])
def test_epilogue_requant_matches_quantizer(plan, opt, B, steps):
    from bflc_demo_b200._native import C
    from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec, sf_bytes
    torch.manual_seed(9)
    spec = mlp_spec(784, 256, 62)
    init = torch.empty(spec.total)
    spec.init_(init, seed=6)
    xu8 = (torch.rand(B * steps, 784, device="cuda") ** 2 * 255).to(torch.uint8)
    y = torch.randint(0, 62, (B * steps,), device="cuda", dtype=torch.int32)
    xb = torch.empty(B * steps, 784, device="cuda", dtype=torch.bfloat16)
    xq = torch.zeros(B * steps, 784, device="cuda", dtype=torch.uint8)
    xsf = torch.full((sf_bytes(B * steps, 784),), 127, device="cuda", dtype=torch.uint8)
    C().prep_inputs(xu8, xb, xq, xsf, 1.0 / 255.0)
    master = init.cuda().clone()
    tr = FlatMLP(spec, master, master.bfloat16(), torch.zeros_like(master), B,
                 lr=(0.05 if opt == "sgd" else 1e-3), optimizer=opt, fp8=True)
    tr.quantize_weights()
    bar = torch.zeros(1, device="cuda", dtype=torch.int32)
    tr.train_epoch_fused(xb, y, steps, bar.data_ptr(), None, plan, 1, x_q=xq, x_sf=xsf)
    torch.cuda.synchronize()
    assert not torch.equal(master, init.cuda())
    got_q, got_dq = tr.work_q.clone(), tr.work_dq.clone()
    tr.quantize_weights()   # the stand-alone quantiser on the trained master
    torch.cuda.synchronize()
    L = tr.ql
    # the weight sections of the blob (its fp32 bias section is written by the quantiser only)
    for name, nbytes in (("w1q", 256 * 784), ("w1sf", 2 * L["kb1"] * 512), ("w2q", 64 * 256),
                         ("w2sf", L["kb2"] * 512)):
        sl = slice(L[name], L[name] + nbytes)
        assert torch.equal(got_q[sl], tr.work_q[sl]), name
    assert torch.equal(got_dq, tr.work_dq)
