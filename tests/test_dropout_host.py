"""Host-side checks of BERT dropout (no GPU):

* a numpy Philox4x32-10 and csrc/include/philox.hpp built with g++ both reproduce the Random123
  known answers, and agree on thousands of keep decisions across seeds, steps, sites and coordinates;
* compiler guard for the dropout instantiations of the tiled attention kernels (build.py's flags):
  present, spill-free, no serialized wgmma, registers recorded; the instantiations without dropout
  keep their register counts;
* PackedTokens.seq_ids: layout and the rebase on slicing;
* run.py --dropout is for BERT only and takes p in [0, 1).

The numpy reference (``keep8_ref``, ``attention_keep_ref``, ``hidden_keep_ref``) is what the GPU
tests compare the device masks against."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from bflc_demo_b200 import build

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK32 = np.uint64(0xFFFFFFFF)
KAT = [  # Random123 known answers: (counter, key) -> output
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


def philox_ref(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on arrays of 32-bit words (any broadcastable shapes) -> 4 uint64 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & MASK32 for x in (c0, c1, c2, c3)]
    k = [np.asarray(x, dtype=np.uint64) & MASK32 for x in (k0, k1)]
    for _ in range(10):
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & MASK32, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & MASK32]
        k = [(k[0] + np.uint64(W0)) & MASK32, (k[1] + np.uint64(W1)) & MASK32]
    return c


def threshold(p: float) -> int:
    """round(p * 65536) in float32 arithmetic, at most 65535 (philox::threshold)."""
    t = np.float32(p) * np.float32(65536.0) + np.float32(0.5)
    return min(int(t) if t > 0 else 0, 65535)


def keep8_ref(seed, step, site, seq, head, row, group, p):
    """The 8 keep bits (bit t = column 8 * group + t) as a uint8 array of the broadcast shape."""
    seed = int(seed)
    w = philox_ref((np.asarray(row, np.uint64) << np.uint64(16)) | np.asarray(group, np.uint64), seq,
                   (np.asarray(site, np.uint64) << np.uint64(8)) | np.asarray(head, np.uint64),
                   np.asarray(step, np.int64).astype(np.uint64) & MASK32, seed & 0xFFFFFFFF, seed >> 32)
    thr = np.uint64(threshold(p))
    bits = np.zeros(np.broadcast(w[0], w[1]).shape, dtype=np.uint8)
    for t in range(8):
        word = w[t >> 1]
        u = (word >> np.uint64(16)) if t & 1 else (word & np.uint64(0xFFFF))
        bits |= ((u >= thr).astype(np.uint8) << np.uint8(t))
    return bits


def _unpack(bits):
    """[..., G] uint8 -> [..., 8 G] bool, column 8 g + t = bit t of group g."""
    return ((bits[..., None] >> np.arange(8, dtype=np.uint8)) & 1).astype(bool).reshape(*bits.shape[:-1], -1)


def attention_keep_ref(seed, step, site, p, B, H, S):
    """Attention keep mask [B*H, S, S] (bool), keyed by (b, h, query row i, key column j)."""
    b, h, i, g = np.meshgrid(np.arange(B), np.arange(H), np.arange(S), np.arange(S // 8), indexing="ij")
    return _unpack(keep8_ref(seed, step, site, b, h, i, g, p)).reshape(B * H, S, S)


def hidden_keep_ref(seed, step, site, p, seq, pos, C):
    """Hidden keep mask [rows, C] (bool) of rows at (seq[r], pos[r])."""
    seq, pos = np.asarray(seq)[:, None], np.asarray(pos)[:, None]
    return _unpack(keep8_ref(seed, step, site, seq, 0, pos, np.arange(C // 8)[None, :], p))


def test_numpy_philox_known_answers():
    for ctr, key, want in KAT:
        got = tuple(int(x) for x in philox_ref(*ctr, *key))
        assert got == want, [f"{x:08x}" for x in got]


HARNESS = r"""
#include <cstdio>
#include "philox.hpp"
using namespace bflc::philox;
int main() {
  unsigned c0, c1, c2, c3, k0, k1;
  while (std::scanf("%u %u %u %u %u %u", &c0, &c1, &c2, &c3, &k0, &k1) == 6) {
    const U4 r = philox4x32_10(U4{c0, c1, c2, c3}, k0, k1);
    std::printf("%u %u %u %u\n", r.x, r.y, r.z, r.w);
  }
  // keep decisions: seed_lo seed_hi step site thr seq head row col
  unsigned s0, s1, st, si, thr, seq, head, row, col;
  while (std::scanf(" k %u %u %u %u %u %u %u %u %u", &s0, &s1, &st, &si, &thr, &seq, &head, &row, &col) == 9) {
    Drop d{s0, s1, st, si, thr, 1.f};
    std::printf("%d\n", keep(d, seq, head, row, col) ? 1 : 0);
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def philox_cpp(tmp_path_factory):
    cxx = os.environ.get("CXX", "g++")
    if shutil.which(cxx) is None:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("philox")
    (d / "h.cpp").write_text(HARNESS)
    exe = d / "h"
    subprocess.run([cxx, "-std=c++17", "-O2", f"-I{build.CSRC / 'include'}", str(d / "h.cpp"), "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    return exe


def test_header_philox_known_answers(philox_cpp):
    inp = "".join(" ".join(str(x) for x in (*ctr, *key)) + "\n" for ctr, key, _ in KAT)
    out = subprocess.run([str(philox_cpp)], input=inp, capture_output=True, text=True, check=True).stdout
    got = [tuple(int(x) for x in ln.split()) for ln in out.splitlines()]
    assert got == [want for _, _, want in KAT]


def test_header_and_numpy_agree_on_keep_decisions(philox_cpp):
    rng = np.random.default_rng(0)
    n = 4000
    seeds = rng.integers(0, 2 ** 63, size=n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=n).astype(np.uint64)
    step = rng.integers(-5, 100000, size=n)
    site = rng.integers(0, 1 << 24, size=n)
    seq = rng.integers(0, 5000, size=n)
    head = rng.integers(0, 256, size=n)
    row = rng.integers(0, 65536, size=n)
    col = rng.integers(0, 8 * 1024, size=n)
    ps = rng.choice([0.1, 0.5, 0.9, 1e-4], size=n)
    lines = ["k " + " ".join(str(int(x)) for x in (int(s) & 0xFFFFFFFF, int(s) >> 32, int(st) & 0xFFFFFFFF, si,
                                                  threshold(p), sq, h, r, c))
             for s, st, si, sq, h, r, c, p in zip(seeds, step, site, seq, head, row, col, ps)]
    out = subprocess.run([str(philox_cpp)], input="\n".join(lines) + "\n", capture_output=True, text=True,
                         check=True).stdout.split()
    cpp = np.array([int(x) for x in out], dtype=bool)
    ref = np.array([(keep8_ref(int(s), st, si, sq, h, r, c >> 3, p) >> (c & 7)) & 1
                    for s, st, si, sq, h, r, c, p in zip(seeds, step, site, seq, head, row, col, ps)], dtype=bool)
    assert len(cpp) == n
    assert np.array_equal(cpp, ref)
    assert 0 < cpp.sum() < n                       # both outcomes occur


def test_threshold_resolution():
    for p in (0.1, 0.5, 1e-3, 0.999, 1 - 2 ** -20):
        assert abs(threshold(p) / 65536 - p) <= 2 ** -16


# ------------------------------------------------------------------------- compiler guard
SRC = build.CSRC / "kernels" / "attn_sm100.cu"
KERNELS = ("attn_fwd_var_kernel", "attn_dq_var_kernel", "attn_dkv_var_kernel")
# registers of every instantiation (kPacked, kDrop), sm_90a with build.py's flags
REGISTERS = {
    (False, False): {"attn_fwd_var_kernel": 128, "attn_dq_var_kernel": 148, "attn_dkv_var_kernel": 154},
    (True, False): {"attn_fwd_var_kernel": 128, "attn_dq_var_kernel": 151, "attn_dkv_var_kernel": 161},
    (False, True): {"attn_fwd_var_kernel": 128, "attn_dq_var_kernel": 168, "attn_dkv_var_kernel": 180},
    (True, True): {"attn_fwd_var_kernel": 128, "attn_dq_var_kernel": 168, "attn_dkv_var_kernel": 180},
}


@pytest.fixture(scope="module")
def ptxas_props(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("no nvcc")
    out = tmp_path_factory.mktemp("ptxas") / "a.o"
    inc = [f"-I{build.CSRC / d}" for d in ("include", "ledger", "runtime")]
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, *inc, "-c", str(SRC), "-o", str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    log = proc.stdout + proc.stderr
    assert proc.returncode == 0, log[-3000:]
    serialized = [ln for ln in log.splitlines() if re.search(r"\(C75(18|20)\)", ln)]
    props = {}
    for name, pk, dr, st, ld, regs in re.findall(
            r"Function properties for \w*?\d(attn_\w+?_var_kernel)ILb([01])ELb([01])E\w*\s*\n\s*"
            r"\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\s*\n"
            r"ptxas info\s*: Used (\d+) registers", log):
        props[(pk == "1", dr == "1", name)] = (int(st), int(ld), int(regs))
    return props, serialized, log


def test_dropout_instantiations_present_spill_free_not_serialized(ptxas_props):
    props, serialized, log = ptxas_props
    assert not serialized, "\n".join(serialized)
    for packed in (False, True):
        for name in KERNELS:
            assert (packed, True, name) in props, log[-3000:]
            st, ld, _ = props[(packed, True, name)]
            assert st == 0 and ld == 0, f"{name} (packed={packed}, dropout): {st} B spill stores / {ld} B loads"


def test_attention_register_counts(ptxas_props):
    props, _, _ = ptxas_props
    for (packed, drop), want in REGISTERS.items():
        got = {name: props[(packed, drop, name)][2] for name in KERNELS}
        assert got == want, f"packed={packed}, dropout={drop}: {got}"


# ------------------------------------------------------------------------- data and CLI
def test_packed_tokens_seq_ids_layout_and_slices():
    from bflc_demo_b200.data.packing import PackedTokens
    lens = [5, 1, 64, 7, 128, 30]
    g = torch.Generator().manual_seed(2)
    x = torch.zeros(len(lens), 128, dtype=torch.int64)
    for i, n in enumerate(lens):
        x[i, :n] = torch.randint(1, 30522, (n,), generator=g)
    pt = PackedTokens.from_padded(x, 0)
    assert pt.seq_ids.dtype == torch.int32
    want = torch.cat([torch.full((n,), i, dtype=torch.int32) for i, n in enumerate(lens)])
    assert torch.equal(pt.seq_ids, want)
    for lo, hi in ((0, 2), (1, 4), (3, 6), (2, 3)):
        s = pt[lo:hi]
        sub = lens[lo:hi]
        assert torch.equal(s.seq_ids, torch.cat([torch.full((n,), i, dtype=torch.int32) for i, n in enumerate(sub)]))
        if len(sub) < 2:
            continue
        s2 = s[1:]                                   # a slice of a slice
        assert torch.equal(s2.seq_ids, torch.cat([torch.full((n,), i, dtype=torch.int32)
                                                  for i, n in enumerate(sub[1:])]))


@pytest.mark.parametrize("args", [["--model", "mlp", "--dropout", "0.1"], ["--model", "resnet18", "--dropout", "0.1"]])
def test_run_rejects_dropout_for_other_models(args, capsys):
    from bflc_demo_b200.run import main
    with pytest.raises(SystemExit) as ei:
        main(args)
    assert ei.value.code == 2
    assert "--dropout" in capsys.readouterr().err


@pytest.mark.parametrize("p", ["1.0", "-0.1", "1.5"])
def test_run_rejects_dropout_outside_unit_interval(p, capsys):
    from bflc_demo_b200.run import main
    with pytest.raises(SystemExit) as ei:
        main(["--model", "bert", "--dropout", p])
    assert ei.value.code == 2
    assert "--dropout" in capsys.readouterr().err


def test_bert_dropout_needs_rng_and_valid_p():
    from bflc_demo_b200.models.nets import BertBase
    with pytest.raises(ValueError):
        BertBase(2, layers=1, dropout=1.0)
    net = BertBase(2, layers=1, dropout=0.1)
    with pytest.raises(ValueError, match="DropoutRNG"):
        net.loss(None, torch.ones(1, 64, dtype=torch.int32), torch.zeros(1, dtype=torch.int32))
    sites = {BertBase.dropout_site(0, k) for k in (BertBase.SITE_EMB, BertBase.SITE_POOL)}
    sites |= {BertBase.dropout_site(i, k) for i in range(12)
              for k in (BertBase.SITE_ATTN, BertBase.SITE_ATTN_OUT, BertBase.SITE_FFN_OUT)}
    assert len(sites) == 2 + 36                     # every site has its own id
