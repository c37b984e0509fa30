"""LoRA across GPUs: scripts/multi_gpu_check.py's ``lora`` mode under torchrun (every visible GPU, >= 2)
fine-tunes rank-8 adapters over a frozen 2-layer GPT for 3 graph-captured rounds; the replicas must
stay bit-identical, the base frozen and every host ledger must agree with the device's.  The
``lora_digest`` mode gives each rank another base: every rank must refuse to build the engine."""
import pytest
import torch

from test_gpu_multi import _run

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def test_lora_multi_gpu_replicas_and_ledgers():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    _, res = _run(["lora"])
    r = res["lora"]
    assert r["epoch"] >= 4 and r["identical"] and r["errs"] == [] and r["chain_ok"] and r["graphs"], r
    assert r["base_frozen"] and r["one_base"] and r["n_params"] == r["adapters"], r


def test_lora_ranks_with_different_bases_are_refused():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    _, res = _run(["lora_digest"])
    assert res["lora_digest"]["refused_everywhere"], res
