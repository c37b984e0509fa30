"""DP-SGD in the persistent MLP trainer across GPUs: scripts/multi_gpu_check.py's ``dpsgd_fused`` mode under
torchrun (every visible GPU, >= 2) runs FusedEngine rounds with ``dpsgd_fused`` and each rank's own secret noise
key; the replicas must stay bit-identical, every host ledger must agree with the device's, and no two ranks
may draw the same noise."""
import pytest
import torch

from test_gpu_multi import _run

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def test_dpsgd_fused_multi_gpu_replicas_ledgers_and_per_rank_noise():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    _, res = _run(["dpsgd_fused"])
    r = res["dpsgd_fused"]
    assert r["epoch"] >= 4 and r["identical"] and r["errs"] == [] and r["chain_ok"] and r["graphs"], r
    assert r["noise_distinct"] and r["dropped"] == 0, r
