"""GPT across GPUs: scripts/multi_gpu_check.py's ``gpt`` mode under torchrun (every visible GPU, >= 2)
trains a 2-layer GPT for 3 graph-captured rounds; the replicas must stay bit-identical and every
host ledger must agree with the device's."""
import pytest
import torch

from test_gpu_multi import _run

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def test_gpt_multi_gpu_replicas_and_ledgers():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    _, res = _run(["gpt"])
    r = res["gpt"]
    assert r["epoch"] >= 4 and r["identical"] and r["errs"] == [] and r["chain_ok"] and r["graphs"], r
