"""DP-SGD across GPUs: scripts/multi_gpu_check.py's ``dpsgd`` mode under torchrun (every visible GPU, >= 2)
runs LoRA GPT rounds with DP-SGD and each rank's own secret noise key; the replicas must stay
bit-identical, every host ledger must agree with the device's, and no two ranks may draw the same noise."""
import pytest
import torch

from test_gpu_multi import _run

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def test_dpsgd_multi_gpu_replicas_ledgers_and_per_rank_noise():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    _, res = _run(["dpsgd"])
    r = res["dpsgd"]
    assert r["epoch"] >= 4 and r["identical"] and r["errs"] == [] and r["chain_ok"] and r["graphs"], r
    assert r["noise_distinct"], r
