"""Plan 4 of the persistent MLP trainer runs fwd1 and the fwd2 -> softmax-xent -> dh chain on 64-row
M-tiles (one 4-CTA cluster per tile), plan 3 on 128-row ones.  Both multiply in the same K order and
the chain epilogue sums each row's exponentials in the same order at either tile height, so after
one step everything that does not go through a float atomic is bit-identical.  Here at batch sizes
that take more clusters than test_gpu_mlp_cluster_chain.py's: B = 1024 is 16 clusters and 64 chain
CTAs, B = 640 leaves plan 3 a half-empty last M-tile that plan 4 fills exactly.  Plan 4's stamps
show that the cluster path ran: it hands its h slice over (slot 1) before its fwd1 epilogue ends
(slot 17), while plan 3 stamps slot 1 after the grid barrier that follows P1."""
import pytest
import torch

from test_gpu_mlp_cluster_chain import _run

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype,opt,B", [("bf16", "adam", 1024), ("fp8", "adam", 1024), ("fp8", "sgd", 640),
                                         ("bf16", "sgd", 640)])
def test_plan4_64row_tiles_match_plan3(dtype, opt, B):
    spec, r3 = _run(3, dtype, opt, B, 1)
    dbg = torch.zeros(1, 32, device="cuda", dtype=torch.int64)
    _, r4 = _run(4, dtype, opt, B, 1, dbg=dbg)
    d = dbg.cpu()
    assert int(d[0, 17]) > 0 and 0 < int(d[0, 1]) <= int(d[0, 17])
    for k in ("h", "dlogits", "dh"):
        assert torch.equal(r4[k], r3[k]), k
    bufs = ("master", "shadow") + (("m", "v") if opt == "adam" else ())
    for buf in bufs:
        v3, v4 = spec.views(r3[buf]), spec.views(r4[buf])
        for k in ("w1", "w2"):
            assert torch.equal(v4[k], v3[k]), (buf, k)
    if dtype == "fp8":
        assert torch.equal(r4["work_q"], r3["work_q"])
        assert torch.equal(r4["work_dq"], r3["work_dq"])
    w0, v3, v4 = spec.views(r3["init"]), spec.views(r3["master"]), spec.views(r4["master"])
    for k in ("b1", "b2"):   # column sums by float atomics: equal up to summation order
        assert torch.allclose(v4[k] - w0[k], v3[k] - w0[k], rtol=1e-4, atol=1e-7), k
    assert abs(r4["loss"] - r3["loss"]) <= 1e-5 * abs(r3["loss"])
    assert r4["correct"] == r3["correct"]
    assert r4["grad_max"] == 0.0
