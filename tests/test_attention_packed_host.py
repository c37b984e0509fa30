"""Host-side checks of packed variable-length BERT (no GPU):

* compiler guard for the packed instantiations of the tiled attention kernels (attn_sm100.cu,
  build.py's flags): present, no serialized wgmma (C7518 / C7520), spill-free;
* PackedTokens: packed ids, positions and cu_seqlens, slicing, and every rejection;
* run.py --packed is for BERT only."""
import os
import re
import shutil
import subprocess

import pytest
import torch

from bflc_demo_b200 import build

SRC = build.CSRC / "kernels" / "attn_sm100.cu"
PACKED = ("attn_fwd_var_kernel", "attn_dq_var_kernel", "attn_dkv_var_kernel")


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("no nvcc")
    out = tmp_path_factory.mktemp("ptxas") / "a.o"
    inc = [f"-I{build.CSRC / d}" for d in ("include", "ledger", "runtime")]
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, *inc, "-c", str(SRC), "-o", str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    log = proc.stdout + proc.stderr
    assert proc.returncode == 0, log[-3000:]
    return log


def test_packed_kernels_present_and_not_serialized(ptxas_log):
    entries = set(re.findall(r"Compiling entry function '\w*?\d(attn_\w+?_kernel)ILb1E", ptxas_log))
    assert entries == set(PACKED), ptxas_log[-3000:]
    serialized = [ln for ln in ptxas_log.splitlines() if re.search(r"\(C75(18|20)\)", ln)]
    assert not serialized, "\n".join(serialized)


def test_packed_kernels_spill_free(ptxas_log):
    props = re.findall(r"Function properties for \w*?\d(attn_\w+?_kernel)ILb1E\w*\s*\n\s*"
                       r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ptxas_log)
    found = {name: (int(st), int(ld)) for name, _, st, ld in props}
    assert set(found) == set(PACKED), ptxas_log[-3000:]
    for name, (st, ld) in found.items():
        assert st == 0 and ld == 0, f"{name} (packed): {st} B spill stores / {ld} B loads"


def _padded(lens, S, pad=0, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.full((len(lens), S), pad, dtype=torch.int64)
    toks = []
    for i, n in enumerate(lens):
        t = torch.randint(1, 30522, (n,), generator=g)
        x[i, :n] = t
        toks.append(t)
    return x, toks


def test_packed_tokens_layout():
    from bflc_demo_b200.data.packing import PackedTokens
    lens = [5, 1, 64, 7, 128]
    x, toks = _padded(lens, 128)
    pt = PackedTokens.from_padded(x, 0)
    assert len(pt) == 5 and pt.T == sum(lens) and pt.max_len == 128
    assert pt.ids.dtype == torch.int32 and pt.pos_ids.dtype == torch.int32 and pt.cu_seqlens.dtype == torch.int32
    assert torch.equal(pt.ids.long(), torch.cat(toks))
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    assert pt.cu_seqlens.tolist() == cu and pt.offsets == cu
    assert torch.equal(pt.pos_ids, torch.cat([torch.arange(n, dtype=torch.int32) for n in lens]))


def test_packed_tokens_slices_rebase():
    from bflc_demo_b200.data.packing import PackedTokens
    lens = [5, 1, 64, 7, 128, 30]
    x, toks = _padded(lens, 128, seed=1)
    pt = PackedTokens.from_padded(x, 0)
    for lo, hi in ((0, 2), (1, 4), (3, 6), (2, 3)):
        s = pt[lo:hi]
        sub = lens[lo:hi]
        assert len(s) == hi - lo and s.T == sum(sub) and s.max_len == max(sub)
        cu = [0]
        for n in sub:
            cu.append(cu[-1] + n)
        assert s.cu_seqlens.tolist() == cu
        assert torch.equal(s.ids.long(), torch.cat(toks[lo:hi]))
        assert torch.equal(s.pos_ids, torch.cat([torch.arange(n, dtype=torch.int32) for n in sub]))
        s2 = s[1:]                                   # a slice of a slice
        assert s2.cu_seqlens.tolist() == [c - cu[1] for c in cu[1:]]
        assert s2.T == sum(sub[1:])
    head = pt[:4]
    assert len(head) == 4 and head.T == sum(lens[:4]) and head.max_len == 64


def test_packed_tokens_rejections():
    from bflc_demo_b200.data.packing import PackedTokens
    x, _ = _padded([5, 0, 3], 64)
    with pytest.raises(ValueError, match="sample 1"):
        PackedTokens.from_padded(x, 0)                 # a sample of length 0
    x, _ = _padded([5, 8], 64)
    x[1, 2] = 0
    with pytest.raises(ValueError, match="right padding"):
        PackedTokens.from_padded(x, 0)                 # pad id inside a sequence
    with pytest.raises(ValueError, match="512"):
        PackedTokens.from_padded(torch.ones(2, 576, dtype=torch.int64), 0)
    with pytest.raises(ValueError):
        from bflc_demo_b200.models.nets import BertBase
        BertBase(2, layers=1, packed=True)             # packed needs a pad id


def test_run_rejects_packed_for_other_models(capsys):
    from bflc_demo_b200.run import main
    with pytest.raises(SystemExit) as ei:
        main(["--model", "mlp", "--packed"])
    assert ei.value.code == 2
    assert "--packed" in capsys.readouterr().err
