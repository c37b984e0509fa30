"""Multi-GPU protocol tests: spawn torchrun over all visible GPUs (>= 2) and assert on the
RESULT line of scripts/multi_gpu_check.py."""
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _run(which, **extra_env):
    n = min(torch.cuda.device_count(), 8)
    n = 8 if n >= 8 else (4 if n >= 4 else 2)
    env = dict(os.environ, PYTHONPATH=ROOT + ":" + os.environ.get("PYTHONPATH", ""), BFLC_NO_AUTOBUILD="1",
               **extra_env)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
                          f"--nproc-per-node={n}", "--master-addr", "127.0.0.1", "--master-port",
                          str(_free_port()), os.path.join(ROOT, "scripts", "multi_gpu_check.py"), *which],
                         capture_output=True, text=True, env=env, timeout=900)
    lines = [l for l in out.stdout.splitlines() if l.startswith("RESULT ")]
    assert lines, out.stdout[-3000:] + out.stderr[-3000:]
    return n, json.loads(lines[0][7:])


def test_fused_engine_multi_gpu():
    n, res = _run(["fused", "two_shot"])
    f = res["fused"]
    assert f["errs"] == [] and f["identical_digest"] and f["identical_chain"] and f["chain_ok"]
    assert all(e == 7 for e in f["epochs"])
    assert f["loss"][-1] < f["loss"][0]
    for mode in res["two_shot"].values():
        assert mode["identical"] and mode["errs"] == [] and mode["chain_ok"]


def test_fedavg_result_equals_weighted_mean_of_uploads():
    """The global model every replica holds == sum_k w_k * upload_k recomputed in PyTorch from the
    trainers' HBM and the host ledger's block (replicas being identical is checked elsewhere;
    this checks they are RIGHT), for the bf16 and the fp8 engine."""
    n, res = _run(["fedavg"])
    for dt in ("bf16", "fp8"):
        r = res["fedavg"][dt]
        assert r["errs"] == [] and r["n_selected"] >= 1
        assert r["worst_rel"] < 1e-6, r          # (bit_exact is reported; fp64 emulation of fma can
                                                 #  double-round a rare element by one ulp)


def test_fused_engine_multi_gpu_fp8():
    """The fused protocol check with MXFP8 candidates: k_pull_blob gathers the trainers' blobs and
    every replica ends on the same digest and chain."""
    n, res = _run(["fused"], BFLC_CHECK_DTYPE="fp8")
    f = res["fused"]
    assert f["errs"] == [] and f["identical_digest"] and f["identical_chain"] and f["chain_ok"]
    assert all(e == 7 for e in f["epochs"]) and f["loss"][-1] < f["loss"][0]


def test_first_k_admission_drops_the_straggler():
    """NEEDED_UPDATE_COUNT < trainers on the device path (C:239-244): with one slow trainer every
    round still completes, exactly K updates are admitted, the slow one is dropped while it is a
    trainer, all replicas agree and the host ledger re-executes every election from the
    admitted mask."""
    n, res = _run(["firstk"])
    if n < 4:
        pytest.skip("first-K admission needs >= 2 trainers: >= 4 GPUs")
    for dt in ("bf16", "fp8"):
        r = res["firstk"][dt]
        assert r["errs"] == [] and r["identical"] and r["chain_ok"] and r["epoch"] == 7
        assert all(a == r["k"] for a in r["admitted_per_round"]), r
        assert r["slow_was_trainer"] >= 5 and r["slow_admitted"] == 0, r


def test_generic_engine_and_byzantine_multi_gpu():
    n, res = _run(["generic", "byzantine"])
    g = res["generic_lenet5"]
    assert g["identical"] and g["errs"] == [] and g["epoch"] == 5
    if n >= 4:
        b = res["byzantine"]
        assert not b["ever_selected"] and not b["ever_elected"]
