"""Compiler guard for the persistent trainer, compiled with build.py's flags (-Xptxas -v):

* its wgmma stay asynchronous: ptxas reports no serialized wgmma (C7518 / C7520) for either
  instantiation of mlp_round_kernel.  Such a warning means a wgmma sits on a path the compiler
  treats as warp-divergent, and every MMA of the kernel then drains before the next one issues;
* its register spills do not grow.  The kernel is not spill-free: the epilogue warpgroups, at
  128 registers per thread, still spill loop state around the per-tile epilogues (DESIGN.md 3.3).
  The ceilings are the byte counts ptxas reports today, so any growth fails here and has to be
  looked at (and the ceilings lowered when a change removes spills)."""
import os
import re
import shutil
import subprocess

import pytest

from bflc_demo_b200 import build

SRC = build.CSRC / "kernels" / "mlp_round_sm100.cu"
# instantiation -> (spill store bytes, spill load bytes) ceilings
SPILL_CEILING = {"ILb0E": (684, 1432),   # bf16
                 "ILb1E": (732, 1408)}   # fp8 (block-scaled MXFP8 forward)


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("no nvcc")
    out = tmp_path_factory.mktemp("ptxas") / "m.o"
    inc = [f"-I{build.CSRC / d}" for d in ("include", "ledger", "runtime")]
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, *inc, "-c", str(SRC), "-o", str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    log = proc.stdout + proc.stderr
    assert proc.returncode == 0, log[-3000:]
    return log


def test_trainer_wgmma_not_serialized(ptxas_log):
    entries = re.findall(r"Compiling entry function '(\w*mlp_round_kernel\w*)'", ptxas_log)
    assert len(entries) == 2, ptxas_log[-3000:]
    serialized = [ln for ln in ptxas_log.splitlines()
                  if re.search(r"\(C75(18|20)\)", ln) and "mlp_round_kernel" in ln]
    assert not serialized, "\n".join(serialized)


def test_trainer_spills_do_not_grow(ptxas_log):
    props = re.findall(r"Function properties for (\w*mlp_round_kernel(ILb[01]E)\w*)\s*\n\s*"
                       r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ptxas_log)
    found = {inst: (int(st), int(ld)) for _, inst, _, st, ld in props}
    assert set(found) == set(SPILL_CEILING), ptxas_log[-3000:]
    for inst, (st, ld) in found.items():
        cs, cl = SPILL_CEILING[inst]
        assert st <= cs and ld <= cl, f"{inst}: {st} B spill stores / {ld} B loads, ceiling {cs} / {cl}"
