"""The bench.py / __graft_entry__.py contract pieces that can be checked without a GPU."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_reports_unavailable_and_exits_zero():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference",
                          "--gpus", "1", "--steps", "3", "--warmup", "3"],
                         capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and isinstance(line["unavailable"], str) and line["unavailable"]


def test_graft_entry_exposes_build_and_smoke():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    assert callable(g.build) and callable(g.smoke)


def test_native_sources_are_all_built_by_build_py():
    """every .cu under csrc is compiled into _C.so (the driver's 'does it build' check covers all)"""
    from bflc_demo_b200 import build as B
    import inspect
    src = inspect.getsource(B)
    assert "kernels" in src and "runtime" in src and "compute_90a" in src and "sm_90a" in src


def test_reference_arm_prints_one_line_under_torchrun():
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", "29577",
                          os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2"],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1 and json.loads(lines[0])["impl"] == "reference"
