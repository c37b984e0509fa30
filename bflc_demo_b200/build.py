"""In-tree native build: nvcc (sm_90a, H100) for the kernel library, g++ for the host runtime.

Produces, next to this file:
  _C.so       CUDA kernels + symmetric-heap runtime + torch bindings
  _ledger.so  C++ ledger runtime (pure host code, pybind11; loads on a CPU-only box)

The ``.so`` files and ``build/`` are git-ignored build products; ``build()`` in
``__graft_entry__.py`` (or ``python -m bflc_demo_b200.build``) (re)builds what is stale.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
OBJ = HERE / "build" / "obj"

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
    "-Xptxas", "-v", "--use_fast_math",
]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function"]


def _torch_paths():
    import torch  # noqa: F401  (slow first import on a fresh box)
    from torch.utils import cpp_extension as ce

    inc = ce.include_paths()
    lib = ce.library_paths()
    return inc, lib


def _run(cmd, log: Path | None = None):
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if log is not None:
        log.write_text(" ".join(map(str, cmd)) + "\n" + proc.stdout + proc.stderr)
    if proc.returncode != 0:
        sys.stderr.write(" ".join(map(str, cmd)) + "\n" + proc.stdout + proc.stderr)
        raise RuntimeError(f"build step failed: {cmd[0]} {cmd[-1]}")
    return proc


def _stale(src: Path, obj: Path, flags: list[str], deps: list[Path]) -> str | None:
    """Returns the new signature when `obj` must be rebuilt, else None."""
    stamp = obj.with_suffix(obj.suffix + ".stamp")
    h = hashlib.sha1(" ".join(flags).encode())
    for d in [src, *deps]:
        h.update(str(d.stat().st_mtime_ns).encode())
    sig = h.hexdigest()
    if obj.exists() and stamp.exists() and stamp.read_text() == sig:
        return None
    stamp.parent.mkdir(parents=True, exist_ok=True)
    stamp.write_text("")  # invalidated until the compile succeeds
    return sig


def _finish(obj: Path, sig: str):
    obj.with_suffix(obj.suffix + ".stamp").write_text(sig)


def build_all(verbose: bool = True) -> dict:
    OBJ.mkdir(parents=True, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cxx = os.environ.get("CXX", "g++")
    py_inc = sysconfig.get_paths()["include"]
    import pybind11

    pyb_inc = pybind11.get_include()
    headers = sorted((CSRC / "include").glob("*")) + sorted((CSRC / "ledger").glob("*.hpp")) + \
        sorted((CSRC / "runtime").glob("*.hpp"))
    inc_flags = [f"-I{CSRC / 'include'}", f"-I{CSRC / 'ledger'}", f"-I{CSRC / 'runtime'}"]

    jobs = []  # (cmd, obj, sig, log)
    objs_c: list[Path] = []
    objs_ledger: list[Path] = []

    # --- CUDA kernels + runtime (.cu): nvcc, no torch headers -> seconds per file
    cu_sources = sorted((CSRC / "kernels").glob("*.cu")) + sorted((CSRC / "runtime").glob("*.cu"))
    for src in cu_sources:
        obj = OBJ / (src.stem + ".o")
        flags = GENCODE + NVCC_FLAGS + inc_flags
        objs_c.append(obj)
        sig = _stale(src, obj, flags, headers)
        if sig:
            jobs.append(([nvcc, *flags, "-c", str(src), "-o", str(obj)], obj, sig,
                         OBJ / (src.stem + ".log")))

    # --- ledger runtime (pure C++)
    for src in sorted((CSRC / "ledger").glob("*.cpp")):
        if src.stem.endswith("_selftest"):      # stand-alone sanitizer driver (has its own main)
            continue
        obj = OBJ / ("ledger_" + src.stem + ".o")
        flags = CXX_FLAGS + inc_flags + [f"-I{py_inc}", f"-I{pyb_inc}"]
        objs_ledger.append(obj)
        sig = _stale(src, obj, flags, headers)
        if sig:
            jobs.append(([cxx, *flags, "-c", str(src), "-o", str(obj)], obj, sig,
                         OBJ / ("ledger_" + src.stem + ".log")))

    # --- torch bindings (g++ with torch headers: the slow one)
    t_inc, t_lib = _torch_paths()
    for src in sorted((CSRC / "bindings").glob("*.cpp")):
        obj = OBJ / ("bind_" + src.stem + ".o")
        flags = CXX_FLAGS + inc_flags + [f"-I{p}" for p in t_inc] + [
            f"-I{py_inc}", "-I/usr/local/cuda/include", "-DTORCH_EXTENSION_NAME=_C",
            "-DTORCH_API_INCLUDE_EXTENSION_H", "-D_GLIBCXX_USE_CXX11_ABI=1", "-Wno-attributes",
        ]
        objs_c.append(obj)
        sig = _stale(src, obj, flags, headers)
        if sig:
            jobs.append(([cxx, *flags, "-c", str(src), "-o", str(obj)], obj, sig,
                         OBJ / ("bind_" + src.stem + ".log")))

    def _do(job):
        cmd, obj, sig, log = job
        if verbose:
            print(f"[build] {Path(cmd[-3]).name}", flush=True)
        _run(cmd, log)
        _finish(obj, sig)

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(_do, jobs))

    suffix = ".so"
    out_c = HERE / ("_C" + suffix)
    out_l = HERE / ("_ledger" + suffix)
    relinked = []
    if jobs or not out_c.exists():
        _run([nvcc, "-shared", *GENCODE, "-o", str(out_c), *map(str, objs_c),
              *[f"-L{p}" for p in t_lib], "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda",
              "-ltorch", "-ltorch_python", "-Xlinker", f"-rpath={t_lib[0]}"])
        relinked.append(out_c.name)
    if jobs or not out_l.exists():
        _run([cxx, "-shared", "-o", str(out_l), *map(str, objs_ledger), "-lpthread"])
        relinked.append(out_l.name)
    return {"compiled": [str(j[1].name) for j in jobs], "linked": relinked}


def ptxas_report() -> str:
    """Concatenated `-Xptxas -v` output of the last compile of every .cu (registers/spills)."""
    out = []
    for log in sorted(OBJ.glob("*.log")):
        txt = log.read_text()
        if "ptxas info" in txt:
            out.append(f"==== {log.stem}\n" + "\n".join(
                ln for ln in txt.splitlines() if "ptxas info" in ln or "Compiling entry" in ln))
    return "\n".join(out)


if __name__ == "__main__":
    res = build_all()
    print(res)
