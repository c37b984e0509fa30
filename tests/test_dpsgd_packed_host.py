"""DP-SGD on packed variable-length BERT, on the host: the dpsgd_packed opt-in and its refusals (config, CLI and
engine), a numpy mirror of the segmented Gram and product-tile norm forms in which each example's value equals
the uniform form on that example alone, bit for bit, and the ptxas report of the segmented kernels."""
import argparse
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from bflc_demo_b200 import build
from bflc_demo_b200.config import FLConfig

F32 = np.float32
LENGTHS = [1, 63, 64, 65, 128, 200, 512]


# ------------------------------------------------------------------ config, CLI and engine
def test_config_accepts_the_opt_in():
    for kw in (dict(lora_rank=8), dict(dpsgd_full_model=True)):
        c = FLConfig(model="bert", dpsgd_clip=1.0, dpsgd_noise=1.0, dpsgd_packed=True, **kw).validate()
        assert c.dpsgd_on and c.dpsgd_packed
    assert not FLConfig().validate().dpsgd_packed


@pytest.mark.parametrize("kw, why", [
    (dict(model="bert", lora_rank=8, dpsgd_packed=True), "dpsgd_packed needs dpsgd_clip > 0"),
    (dict(model="gpt", lora_rank=8, dpsgd_clip=1.0, dpsgd_packed=True), "applies to packed bert, not gpt"),
    (dict(model="mlp", dpsgd_clip=1.0, dpsgd_packed=True), "applies to packed bert, not mlp"),
    (dict(model="bert", lora_rank=8, dpsgd_clip=1.0, dpsgd_packed=True, samples_per_client=64, batch_size=16,
          dpsgd_sampling="poisson"), "needs dpsgd_sampling='partition'"),
    (dict(model="bert", lora_rank=8, dpsgd_clip=1.0, dpsgd_packed=True, dpsgd_conv=True), "dpsgd_conv"),
    (dict(model="bert", lora_rank=8, dpsgd_clip=1.0, dpsgd_packed=True, dpsgd_fused=True), "dpsgd_fused"),
])
def test_config_refuses(kw, why):
    with pytest.raises(ValueError, match=re.escape(why)):
        FLConfig(**kw).validate()


def _cli_fields(argv):
    from bflc_demo_b200 import run
    ap = argparse.ArgumentParser()
    for flag in ("--packed", "--generic"):
        ap.add_argument(flag, action="store_true")
    ap.add_argument("--model", default="bert")
    ap.add_argument("--dtype", default="bf16")
    ap.add_argument("--lora-rank", type=int, default=0)
    ap.add_argument("--resnet-norm", default=None)
    run.add_dpsgd_args(ap)
    return run.dpsgd_fields(ap, ap.parse_args(argv))


def test_cli_accepts_the_opt_in():
    kw = _cli_fields(["--packed", "--lora-rank", "8", "--dpsgd-clip", "1", "--dpsgd-noise", "1", "--dpsgd-packed"])
    assert kw["dpsgd_packed"] and kw["dpsgd_clip"] == 1
    assert _cli_fields(["--packed", "--dpsgd-clip", "1", "--dpsgd-full-model", "--dpsgd-packed"])["dpsgd_packed"]


@pytest.mark.parametrize("argv, why", [
    (["--model", "bert", "--lora-rank", "8", "--packed", "--dpsgd-packed"], "--dpsgd-packed needs --dpsgd-clip"),
    (["--model", "bert", "--lora-rank", "8", "--dpsgd-clip", "1", "--dpsgd-packed"], "--dpsgd-packed needs --packed"),
    (["--model", "bert", "--lora-rank", "8", "--packed", "--dpsgd-clip", "1", "--dpsgd-packed", "--dpsgd-sampling",
      "poisson"], "needs dpsgd_sampling='partition'"),
    # without the opt-in the refusal stands, naming it
    (["--model", "bert", "--lora-rank", "8", "--packed", "--dpsgd-clip", "1"], "does not support --packed"),
    (["--model", "bert", "--lora-rank", "8", "--packed", "--dpsgd-clip", "1"], "--dpsgd-packed"),
])
def test_cli_refuses(argv, why, capsys):
    from bflc_demo_b200.run import main
    with pytest.raises(SystemExit) as e:
        main(argv)
    assert e.value.code == 2
    assert why in capsys.readouterr().err


@pytest.mark.parametrize("case", ["packed_without_opt_in", "opt_in_padded_bert", "opt_in_mlp"])
def test_engine_refuses_before_touching_the_device(case):
    """GenericFedEngine's refusals run before any device work, so they hold without a GPU."""
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import BertBase, MLPNet
    kw = dict(model="bert", lora_rank=0, dpsgd_clip=1.0, dpsgd_full_model=True, clients=1, committee_size=1,
              needed_updates=1, aggregate_count=1, solo=True)
    if case == "packed_without_opt_in":
        cfg, net, why = FLConfig(**kw).validate(), BertBase(2, layers=1, pad_id=0, packed=True), "packed batches"
    elif case == "opt_in_padded_bert":
        cfg, net, why = FLConfig(dpsgd_packed=True, **kw).validate(), BertBase(2, layers=1, pad_id=0), "packed BertBase"
    else:
        cfg = FLConfig(dpsgd_clip=1.0, dpsgd_packed=False, clients=1, committee_size=1, needed_updates=1,
                       aggregate_count=1, solo=True).validate()
        cfg.dpsgd_packed = True      # past validate(), as a caller that mutates a config would
        net, why = MLPNet(), "packed BertBase"
    try:
        GenericFedEngine(cfg, net, shard=None)
    except ValueError as e:
        assert why in str(e)
    else:
        pytest.fail("not refused")


# ------------------------------------------------------------------ numpy mirror of the segmented forms
def _pairs(tiles, sym=True):
    """The kernel's pair decode: blockIdx.x -> (ti, tj)."""
    out = []
    for p in range(tiles * (tiles + 1) // 2 if sym else tiles * tiles):
        ti, tj = 0, p
        if sym:
            while tj >= tiles - ti:
                tj -= tiles - ti
                ti += 1
            tj += ti
        else:
            ti, tj = tj // tiles, tj % tiles
        out.append((ti, tj))
    return out


def _tile(X, row0, n):
    """64 rows of X from row0, rows past n zero-filled (gram_acc's loads)."""
    t = np.zeros((64, X.shape[1]), F32)
    t[:n] = X[row0:row0 + n]
    return t


def _pair_partial(P, Q, bias, row0, R, ti, tj):
    ni, nj = min(64, R - 64 * ti), min(64, R - 64 * tj)
    gp = (_tile(P, row0 + 64 * ti, ni) @ _tile(P, row0 + 64 * tj, nj).T).astype(F32)
    gq = ((_tile(Q, row0 + 64 * ti, ni) @ _tile(Q, row0 + 64 * tj, nj).T).astype(F32) + F32(bias)).astype(F32)
    s = F32((gp * gq).astype(F32).sum(dtype=F32))
    return s if ti == tj else F32(2) * s


def gram_uniform(P, Q, bias, R, B):
    """k_pe_gram: out [pairs(R), B]."""
    pr = _pairs((R + 63) // 64)
    out = np.zeros((len(pr), B), F32)
    for n in range(B):
        for k, (ti, tj) in enumerate(pr):
            out[k, n] = _pair_partial(P, Q, bias, n * R, R, ti, tj)
    return out


def gram_segmented(P, Q, bias, cu, max_len, start=None):
    """k_packed_gram: pairs of ceil(max_len / 64) tiles; a pair past the example's own tiles is +0.  ``start``
    (a modelled mistake) overrides where an example's rows begin."""
    B = len(cu) - 1
    pr = _pairs((max_len + 63) // 64)
    out = np.zeros((len(pr), B), F32)
    for n in range(B):
        row0, L = (cu[n] if start is None else start(n)), cu[n + 1] - cu[n]
        for k, (ti, tj) in enumerate(pr):
            if 64 * ti < L and 64 * tj < L:
                out[k, n] = _pair_partial(P, Q, bias, row0, L, ti, tj)
    return out


def tiles_uniform(A, Bm, R, B):
    """k_pe_norm over a single 64 x 64 column tile: per example, the K loop over its R rows in 64-row chunks."""
    out = np.zeros(B, F32)
    for n in range(B):
        d = np.zeros((A.shape[1], Bm.shape[1]), F32)
        for t0 in range(0, R, 64):
            d = (d + (_tile(A, n * R + t0, min(64, R - t0)).T @ _tile(Bm, n * R + t0, min(64, R - t0))).astype(F32))
        out[n] = (d * d).astype(F32).sum(dtype=F32)
    return out


def tiles_segmented(A, Bm, cu, rows_of=None):
    B = len(cu) - 1
    out = np.zeros(B, F32)
    for n in range(B):
        row0, L = cu[n], (cu[n + 1] - cu[n] if rows_of is None else rows_of(n))
        d = np.zeros((A.shape[1], Bm.shape[1]), F32)
        for t0 in range(0, L, 64):
            d = (d + (_tile(A, row0 + t0, min(64, L - t0)).T @ _tile(Bm, row0 + t0, min(64, L - t0))).astype(F32))
        out[n] = (d * d).astype(F32).sum(dtype=F32)
    return out


def _fixture(width_p, width_q, seed=0):
    rng = np.random.default_rng(seed)
    cu = np.concatenate([[0], np.cumsum(LENGTHS)]).astype(np.int64)
    T = int(cu[-1])
    # integers scaled by 2^-4: fp32 products and sums of these stay exact, so the fp64 check can be tight
    P = (rng.integers(-3, 4, (T, width_p)) / 16).astype(F32)
    Q = (rng.integers(-3, 4, (T, width_q)) / 16).astype(F32)
    return cu, P, Q


def _clip_sum(col):
    """k_dpsgd_clip's fp32 sum of one example's rows, in row order."""
    s = F32(0)
    for v in col:
        s = F32(s + v)
    return s


def test_segmented_gram_equals_each_example_alone_bit_for_bit():
    cu, P, Q = _fixture(8, 12)
    seg = gram_segmented(P, Q, 1.0, cu, max(LENGTHS))
    assert seg.shape == (36, len(LENGTHS))
    for n, L in enumerate(LENGTHS):
        alone = gram_uniform(P[cu[n]:cu[n + 1]], Q[cu[n]:cu[n + 1]], 1.0, L, 1)[:, 0]
        assert _clip_sum(seg[:, n]).view(np.uint32) == _clip_sum(alone).view(np.uint32), L
        # and it is the example's ||P_n^T [Q_n | 1]||^2
        Qn = np.concatenate([Q[cu[n]:cu[n + 1]], np.ones((L, 1), F32)], 1).astype(np.float64)
        ref = np.square(P[cu[n]:cu[n + 1]].astype(np.float64).T @ Qn).sum()
        assert abs(float(_clip_sum(seg[:, n])) - ref) <= 1e-6 * ref, (L, ref)


def test_segmented_product_tiles_equal_each_example_alone_bit_for_bit():
    cu, A, Bm = _fixture(64, 8, seed=1)
    seg = tiles_segmented(A, Bm, cu)
    for n, L in enumerate(LENGTHS):
        alone = tiles_uniform(A[cu[n]:cu[n + 1]], Bm[cu[n]:cu[n + 1]], L, 1)[0]
        assert seg[n].view(np.uint32) == alone.view(np.uint32), L
        ref = np.square(A[cu[n]:cu[n + 1]].astype(np.float64).T @ Bm[cu[n]:cu[n + 1]].astype(np.float64)).sum()
        assert abs(float(seg[n]) - ref) <= 1e-6 * ref, L


def test_fixture_catches_uniform_offsets_and_unmasked_tails():
    """Modelled mistakes: an example's rows taken from n * max_len (the uniform layout), or its last tile read
    to 64 rows (the next example's tokens): both change some example's norm."""
    cu, P, Q = _fixture(8, 12)
    good = gram_segmented(P, Q, 0.0, cu, max(LENGTHS))
    T = int(cu[-1])
    Pz, Qz = np.zeros((len(LENGTHS) * 512, 8), F32), np.zeros((len(LENGTHS) * 512, 12), F32)
    Pz[:T], Qz[:T] = P, Q
    wrong = gram_segmented(Pz, Qz, 0.0, cu, max(LENGTHS), start=lambda n: n * 512)
    assert not np.array_equal(good, wrong)
    cu2, A, Bm = _fixture(64, 8, seed=1)
    tiles = tiles_segmented(A, Bm, cu2)
    Ap, Bp = np.concatenate([A, np.zeros((64, 64), F32)]), np.concatenate([Bm, np.zeros((64, 8), F32)])
    padded = tiles_segmented(Ap, Bp, cu2, rows_of=lambda n: -(-(cu2[n + 1] - cu2[n]) // 64) * 64)
    assert not np.array_equal(tiles, padded)


# ------------------------------------------------------------------ ptxas
def _ptxas(tmp_path, name):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(nvcc).exists():
        pytest.skip("nvcc not found")
    src = Path(build.CSRC) / "kernels" / name
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, "-I", str(Path(build.CSRC) / "include"), "-c", str(src),
           "-o", str(tmp_path / "k.o")]
    out = subprocess.run(cmd, capture_output=True, text=True, check=True)
    log = out.stdout + out.stderr
    return {name: props for name, *props in re.findall(
        r"Function properties for (\w+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
        log)}


def test_segmented_kernels_ptxas_clean(tmp_path):
    """Every segmented instantiation (k_packed_*): no stack frame, no spills."""
    props = _ptxas(tmp_path, "dpsgd_kernels.cu")
    for k in ("k_packed_norm", "k_packed_gram", "k_packed_rows", "k_packed_ln", "k_packed_ln_release",
              "k_packed_scale_rows"):
        hits = [p for name, p in props.items() if re.search(rf"\d{k}E", name)]
        assert len(hits) == 1, (k, sorted(props))
        assert hits[0] == ["0", "0", "0"], (k, hits[0])
