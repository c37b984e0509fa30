"""FedProx with two or more ranks (``scripts/multi_gpu_check.py prox`` under torchrun): each rank's
anchor is its own replica of the global model, which the peers' consensus kernels rewrite.  After
three rounds of the fused engine (bf16 and MXFP8) and of the generic engine (LeNet-5 with a recipe),
every replica holds the same global model bit for bit and every host ledger re-executes with no
mismatch."""
import pytest

from test_gpu_multi import _run

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def test_prox_replicas_stay_identical_and_ledgers_agree():
    n, res = _run(["prox"])
    for name in ("fused_bf16", "fused_fp8", "generic_lenet5"):
        r = res["prox"][name]
        assert r["anchored"] and r["identical"] and r["errs"] == [] and r["chain_ok"], (name, r)
        assert r["epochs"] == [3] * n, (name, r)
