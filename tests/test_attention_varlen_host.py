"""Host-side checks of padded variable-length BERT (no GPU):

* compiler guard for attn_sm100.cu, compiled with build.py's flags (-Xptxas -v): no attention
  kernel runs serialized wgmma (C7518 / C7520), the tiled forward and backward kernels are
  spill-free;
* tokens_like(min_len=...) produces right-padded samples, and its default output is unchanged;
* BertBase rejects sequences longer than its position table;
* run.py rejects a --seq-len the fused attention kernels cannot take."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from bflc_demo_b200 import build

SRC = build.CSRC / "kernels" / "attn_sm100.cu"
# kernel -> (spill store bytes, spill load bytes) ceilings
SPILL_CEILING = {"attn_fwd_var_kernel": (0, 0),
                 "attn_dq_var_kernel": (0, 0),
                 "attn_dkv_var_kernel": (0, 0)}


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


def test_attention_wgmma_not_serialized(ptxas_log):
    entries = re.findall(r"Compiling entry function '\w*?\d(attn_[a-z]+(?:_var)?_kernel)", ptxas_log)
    assert set(SPILL_CEILING) <= set(entries), ptxas_log[-3000:]
    serialized = [ln for ln in ptxas_log.splitlines() if re.search(r"\(C75(18|20)\)", ln)]
    assert not serialized, "\n".join(serialized)


def test_tiled_attention_spills(ptxas_log):
    props = re.findall(r"Function properties for \w*?\d(attn_[a-z]+(?:_var)?_kernel)\w*\s*\n\s*"
                       r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ptxas_log)
    found = {name: (int(st), int(ld)) for name, _, st, ld in props if name in SPILL_CEILING}
    assert set(found) == set(SPILL_CEILING), ptxas_log[-3000:]
    for name, (st, ld) in found.items():
        cs, cl = SPILL_CEILING[name]
        assert st <= cs and ld <= cl, f"{name}: {st} B spill stores / {ld} B loads, ceiling {cs} / {cl}"


def test_tokens_like_min_len_right_pads():
    from bflc_demo_b200.data.synthetic import tokens_like
    seq, lo, pad = 128, 40, 0
    shards = tokens_like(3, 64, seed=5, seq_len=seq, min_len=lo, pad_id=pad)
    seen = set()
    for sh in shards:
        x = sh.x.numpy()
        assert x.shape == (64, seq)
        lengths = (x != pad).sum(1)
        assert lengths.min() >= lo and lengths.max() <= seq
        # pad_id only as a suffix: every position before the length is a real token
        assert ((np.arange(seq)[None, :] < lengths[:, None]) == (x != pad)).all()
        seen.update(lengths.tolist())
    assert len(seen) > 10                     # lengths actually vary
    assert (tokens_like(1, 64, seed=5, seq_len=seq, min_len=lo, pad_id=7)[0].x != 7).sum(1).min() >= lo
    with pytest.raises(ValueError):
        tokens_like(1, 4, seq_len=seq, min_len=seq + 1)


def test_tokens_like_default_unchanged():
    from bflc_demo_b200.data.synthetic import tokens_like
    a = tokens_like(2, 16, seed=9)
    b = tokens_like(2, 16, seed=9, min_len=None)
    for sa, sb in zip(a, b):
        assert torch.equal(sa.x, sb.x) and torch.equal(sa.y, sb.y)


def test_bert_rejects_sequences_longer_than_positions():
    from bflc_demo_b200.models.nets import BertBase
    net = BertBase(2, layers=1, pad_id=0)
    with pytest.raises(ValueError, match="position"):
        net.features(None, torch.ones(1, 576, dtype=torch.int32), False)


@pytest.mark.parametrize("args", [["--seq-len", "100"], ["--seq-len", "576"], ["--seq-len", "0"],
                                  ["--seq-len", "256", "--min-seq-len", "300"],
                                  ["--seq-len", "256", "--min-seq-len", "0"]])
def test_run_rejects_bad_seq_len(args, capsys):
    from bflc_demo_b200.run import main
    with pytest.raises(SystemExit) as ei:
        main(["--model", "bert", *args])
    assert ei.value.code == 2
    assert "seq-len" in capsys.readouterr().err
