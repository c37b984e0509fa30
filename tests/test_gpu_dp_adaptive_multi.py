"""Adaptive clipping over 2+ GPUs: scripts/multi_gpu_check.py dp_adaptive -- replicas bit-identical, every
clip record and model equal to the oracle's, and every host ledger re-executing the clip trajectory."""
from __future__ import annotations

import json
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]


@pytest.mark.gpu
def test_multi_gpu_dp_adaptive_check():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs 2 GPUs")
    n = min(n, 8)
    cmd = [sys.executable, "-m", "torch.distributed.run", f"--nproc_per_node={n}",
           str(ROOT / "scripts" / "multi_gpu_check.py"), "dp_adaptive"]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1800,
                       env=dict(os.environ, PYTHONPATH=str(ROOT)))
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    line = [ln for ln in p.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    res = json.loads(line[len("RESULT "):])["dp_adaptive"]
    for name, r in res.items():
        assert r["errs"] == [] and r["identical"] and r["bit_exact"] and r["clip_ok"], (name, r)
        assert r["clips"][-1] > r["clips"][0], (name, r["clips"])      # from 100x too small, the clip grows
