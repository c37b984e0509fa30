"""Host-side checks of the causal language-modelling work: the topic-mixture corpus, run.py's gpt flags,
an fp64 GPT reference against stock torch modules, and the compiler guard of the causal attention
kernels.  No GPU needed."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from bflc_demo_b200 import build
from bflc_demo_b200.data.synthetic import lm_corpus_like


# ------------------------------------------------------------------------------- corpus
def test_corpus_deterministic_and_only_matches_full():
    a = lm_corpus_like(3, 16, seed=5, seq_len=64, vocab=1000)
    b = lm_corpus_like(3, 16, seed=5, seq_len=64, vocab=1000)
    for sa, sb in zip(a, b):
        assert torch.equal(sa.x, sb.x) and torch.equal(sa.y, sb.y)
    for i in range(3):
        one = lm_corpus_like(3, 16, seed=5, seq_len=64, vocab=1000, only=i)
        assert len(one) == 1 and torch.equal(one[0].x, a[i].x) and torch.equal(one[0].y, a[i].y)
    assert not torch.equal(a[0].x, a[1].x)
    c = lm_corpus_like(1, 16, seed=6, seq_len=64, vocab=1000)[0]
    assert not torch.equal(c.x, a[0].x)


def test_corpus_shift_and_range():
    sh = lm_corpus_like(2, 32, seed=1, seq_len=128, vocab=777)[1]
    assert sh.x.shape == sh.y.shape == (32, 128) and sh.x.dtype == sh.y.dtype == torch.int64
    assert torch.equal(sh.y[:, :-1], sh.x[:, 1:])
    assert int(sh.x.min()) >= 0 and int(sh.y.max()) < 777 and sh.n_classes == 777
    assert len(sh) == 32


def _topics_of(shard, seed, vocab, topics, successors=4):
    """Each sample's topic: the table whose successor sets explain most of its transitions."""
    succ = np.random.default_rng([seed, 77]).integers(0, vocab, size=(topics, vocab, successors))
    x, y = shard.x.numpy(), shard.y.numpy()
    hits = np.stack([(succ[t][x] == y[..., None]).any(-1).sum(-1) for t in range(topics)], -1)
    return hits.argmax(-1)


def test_topic_skew():
    V, T, n = 512, 8, 400
    iid = lm_corpus_like(2, n, seed=3, seq_len=64, vocab=V, topics=T, alpha=0.0)
    for sh in iid:
        hist = np.bincount(_topics_of(sh, 3, V, T), minlength=T) / n
        assert np.abs(hist - 1 / T).max() < 0.07           # near uniform
    skew = lm_corpus_like(2, n, seed=3, seq_len=64, vocab=V, topics=T, alpha=0.1)
    h = [np.bincount(_topics_of(sh, 3, V, T), minlength=T) / n for sh in skew]
    assert max(x.max() for x in h) > 0.4                   # Dirichlet(0.1): a dominant topic
    assert np.abs(h[0] - h[1]).sum() > 0.5                  # and the clients differ


# ------------------------------------------------------------------------------ run.py
@pytest.mark.parametrize("argv", [
    ["--model", "gpt", "--min-seq-len", "64"],
    ["--model", "gpt", "--packed"],
    ["--model", "gpt", "--seq-len", "100"],
    ["--model", "gpt", "--dropout", "1.0"],
    ["--model", "lenet5", "--dropout", "0.1"],
])
def test_run_rejects_gpt_flag_combinations(argv):
    from bflc_demo_b200 import run
    with pytest.raises(SystemExit) as e:
        run.main(argv + ["--rounds", "1"])
    assert e.value.code == 2


# ------------------------------------------------------------------- fp64 GPT reference
def ref_gpt(P, ids, L, H, eps=1e-12):
    """Independent fp64 pre-LN GPT-2 forward -> logits [N*S, V] (what the GPU conformance suite uses)."""
    B, S = ids.shape
    Hd = P["emb.word"].shape[1]
    x = P["emb.word"][ids.reshape(-1)] + P["emb.pos"][torch.arange(S).repeat(B)]

    def ln(x, p):
        mu = x.mean(-1, keepdim=True)
        var = ((x - mu) ** 2).mean(-1, keepdim=True)
        return (x - mu) / torch.sqrt(var + eps) * P[p + ".gamma"] + P[p + ".beta"]

    def lin(x, p):
        return x @ P[p + ".w"].T + P[p + ".b"]

    for i in range(L):
        pf = f"dec{i}"
        a = ln(x, f"{pf}.ln1")
        q, k, v = (lin(a, f"{pf}.{n}").view(B, S, H, Hd // H).transpose(1, 2) for n in "qkv")
        s = (q @ k.mT) / (Hd // H) ** 0.5
        s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool).tril(), float("-inf"))
        att = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B * S, Hd)
        x = x + lin(att, f"{pf}.o")
        x = x + lin(torch.nn.functional.gelu(lin(ln(x, f"{pf}.ln2"), f"{pf}.ff1")), f"{pf}.ff2")
    return ln(x, "ln_f") @ P["emb.word"].T


def test_fp64_gpt_matches_stock_torch():
    from bflc_demo_b200.models.nets import GPT
    L, Hd, H, V, S, B = 2, 128, 2, 300, 64, 3
    net = GPT(layers=L, hidden=Hd, heads=H, ffn=256, vocab=V, max_pos=S)
    flat = torch.empty(net.spec.total, dtype=torch.float32)
    net.init_(flat, seed=4)
    P = {k: t.double() for k, t in net.spec.views(flat).items()}
    for k in P:                                   # non-trivial vectors
        if not k.endswith(".w") and k not in ("emb.word", "emb.pos"):
            P[k] = P[k] + 0.1 * torch.randn(P[k].shape, dtype=torch.float64)
    ids = torch.randint(0, V, (B, S))
    ref = ref_gpt(P, ids, L, H)

    emb = torch.nn.Embedding(V, Hd).double()
    pos = torch.nn.Embedding(S, Hd).double()
    emb.weight.data, pos.weight.data = P["emb.word"], P["emb.pos"]
    x = emb(ids) + pos(torch.arange(S))[None]
    for i in range(L):
        pf = f"dec{i}"
        mods = {}
        for nm in ("ln1", "ln2"):
            m = torch.nn.LayerNorm(Hd, eps=1e-12).double()
            m.weight.data, m.bias.data = P[f"{pf}.{nm}.gamma"], P[f"{pf}.{nm}.beta"]
            mods[nm] = m
        for nm, (o, i_) in dict(q=(Hd, Hd), k=(Hd, Hd), v=(Hd, Hd), o=(Hd, Hd), ff1=(256, Hd), ff2=(Hd, 256)).items():
            m = torch.nn.Linear(i_, o).double()
            m.weight.data, m.bias.data = P[f"{pf}.{nm}.w"], P[f"{pf}.{nm}.b"]
            mods[nm] = m
        a = mods["ln1"](x)
        q, k, v = (mods[n](a).view(B, S, H, Hd // H).transpose(1, 2) for n in "qkv")
        att = torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True)
        x = x + mods["o"](att.transpose(1, 2).reshape(B, S, Hd))
        x = x + mods["ff2"](torch.nn.functional.gelu(mods["ff1"](mods["ln2"](x))))
    lnf = torch.nn.LayerNorm(Hd, eps=1e-12).double()
    lnf.weight.data, lnf.bias.data = P["ln_f.gamma"], P["ln_f.beta"]
    logits = lnf(x).reshape(B * S, Hd) @ emb.weight.T
    assert torch.allclose(ref, logits, atol=1e-10, rtol=1e-10)


def test_gpt_spec_and_build_model():
    from bflc_demo_b200.models.nets import GPT, build_model
    net = build_model("gpt", 8192, layers=2)
    assert isinstance(net, GPT) and net.n_classes == 8192 and net.L == 2
    names = net.spec.by_name
    assert "emb.word" in names and "ln_f.gamma" in names and "dec1.ff2.w" in names
    assert not any(k.startswith("cls") or k.startswith("fc") for k in names)     # the head is tied
    with pytest.raises(ValueError):
        GPT(hidden=100, heads=2)
    with pytest.raises(ValueError):
        GPT(dropout=1.0)
    assert GPT.dropout_site(3, GPT.SITE_FFN_OUT) == 27


# ----------------------------------------------------------------------- compiler guard
def test_causal_attention_kernels_spill_free(tmp_path):
    """Every tiled attention instantiation, the causal ones included, compiles for sm_90a with zero
    spill bytes and no serialized wgmma."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("no nvcc")
    inc = [f"-I{build.CSRC / d}" for d in ("include", "ledger", "runtime")]
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, *inc, "-c", str(build.CSRC / "kernels" / "attn_sm100.cu"),
           "-o", str(tmp_path / "a.o")]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    log = proc.stdout + proc.stderr
    assert proc.returncode == 0, log[-3000:]
    assert not [ln for ln in log.splitlines() if re.search(r"\(C75(18|20)\)", ln)]
    props = re.findall(r"Function properties for \w*?\d(attn_(?:causal_\w+?|\w+?_var_kernel)I\w+?E)\w*\s*\n\s*"
                       r"\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    found = {name for name, _, _ in props}
    want = {f"attn_causal_{k}ILb{d}E" for k in ("fwd", "dq", "dkv") for d in (0, 1)}
    assert want <= found, sorted(found)
    assert len(props) == 6 + 12, sorted(found)          # 6 causal + 3 kernels x (kPacked, kDrop)
    for name, st, ld in props:
        assert st == "0" and ld == "0", f"{name}: {st} B spill stores / {ld} B spill loads"
