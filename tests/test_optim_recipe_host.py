"""Host-side checks of the fine-tuning optimizer recipe (no GPU):

* the no-decay mask covers exactly the 1-D entries of LeNet-5, ResNet-18 and BERT-base;
* the host lr factor equals an independent transcription of the HF schedule lambdas;
* FLConfig and run.py reject bad recipe values, and run.py rejects the recipe with the fused MLP engine;
* compiler guard (build.py's flags): the recipe instantiations of k_optim and the norm kernel are present
  and spill-free, and the plain SGD / Adam instantiations keep their register counts."""
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from bflc_demo_b200 import build
from bflc_demo_b200.config import FLConfig


# ------------------------------------------------------------------------- mask
def _specs():
    from bflc_demo_b200.models.nets import BertBase, LeNet5, ResNet18
    return {"lenet5": LeNet5(10).spec, "resnet18": ResNet18(10).spec, "bert": BertBase(2).spec}


def _bits(mask, n):
    words = mask.numpy().view(np.uint32)
    blocks = ((words[:, None] >> np.arange(32, dtype=np.uint32)) & 1).astype(bool).reshape(-1)
    return np.repeat(blocks, 8)[:n]          # per float


@pytest.mark.parametrize("name", ["lenet5", "resnet18", "bert"])
def test_no_decay_mask_covers_exactly_the_vectors(name):
    from bflc_demo_b200.ops.optim import no_decay_mask
    spec = _specs()[name]
    mask = no_decay_mask(spec)
    assert mask.dtype == torch.int32 and mask.numel() == (spec.total + 255) // 256
    per_float = _bits(mask, spec.total)
    n_vec = 0
    for e in spec.entries:
        got = per_float[e.offset:e.offset + e.numel]
        if len(e.shape) == 1:
            assert got.all(), e.name
            n_vec += 1
        else:
            assert not got.any(), e.name
    assert n_vec > 0
    if name == "resnet18":                    # batch-norm running statistics are never decayed
        assert any(e.name.endswith("rmean") for e in spec.entries)


def test_no_decay_mask_other_lengths():
    from bflc_demo_b200.models.flat import ParamSpec
    from bflc_demo_b200.ops.optim import no_decay_mask
    spec = ParamSpec([("w", (3, 5)), ("b", (3,)), ("g", (9,)), ("w2", (4, 4))])
    assert [e.offset for e in spec.entries] == [0, 16, 24, 40]
    per_float = _bits(no_decay_mask(spec), spec.total)
    assert not per_float[:16].any() and per_float[16:40].all() and not per_float[40:56].any()
    assert no_decay_mask(spec, 1000).numel() == 4


# ------------------------------------------------------------------------- schedule
def hf_lambda(schedule, W, T):
    """The lambdas of transformers.get_{constant,linear,cosine}_schedule_with_warmup (num_cycles 0.5)."""
    def constant(step):
        if step < W:
            return float(step) / float(max(1.0, W))
        return 1.0

    def linear(step):
        if step < W:
            return float(step) / float(max(1, W))
        return max(0.0, float(T - step) / float(max(1, T - W)))

    def cosine(step):
        if step < W:
            return float(step) / float(max(1, W))
        progress = float(step - W) / float(max(1, T - W))
        return max(0.0, 0.5 * (1.0 + math.cos(math.pi * float(0.5) * 2.0 * progress)))
    return dict(constant=constant, linear=linear, cosine=cosine)[schedule]


@pytest.mark.parametrize("schedule", ["constant", "linear", "cosine"])
@pytest.mark.parametrize("W,T", [(0, 10), (3, 10), (1, 2), (10, 1000)])
def test_host_lr_factor_matches_hf(schedule, W, T):
    from bflc_demo_b200.ops.optim import lr_factor
    ref = hf_lambda(schedule, W, T)
    for s in sorted({0, max(W - 1, 0), W, T - 1, T, T + 5}):
        assert lr_factor(schedule, s, W, T) == pytest.approx(ref(s), rel=1e-12, abs=1e-15), (s, W, T)


# ------------------------------------------------------------------------- config and CLI
@pytest.mark.parametrize("kw", [dict(weight_decay=-0.1), dict(lr_schedule="step"), dict(warmup_steps=-1),
                                dict(total_steps=-5), dict(clip_grad_norm=-1.0),
                                dict(lr_schedule="linear", warmup_steps=5, total_steps=5),
                                dict(lr_schedule="cosine", total_steps=0), dict(weight_decay=float("nan"))])
def test_config_rejects_bad_recipe(kw):
    with pytest.raises(ValueError):
        FLConfig(**kw).validate()


def test_config_recipe_defaults_and_env(monkeypatch):
    c = FLConfig().validate()
    assert not c.has_optim_recipe
    assert FLConfig(lr_schedule="constant", warmup_steps=3).validate().has_optim_recipe
    monkeypatch.setenv("BFLC_WEIGHT_DECAY", "0.01")
    monkeypatch.setenv("BFLC_LR_SCHEDULE", "cosine")
    monkeypatch.setenv("BFLC_TOTAL_STEPS", "100")
    monkeypatch.setenv("BFLC_CLIP_GRAD_NORM", "1.0")
    e = FLConfig.from_env()
    assert (e.weight_decay, e.lr_schedule, e.total_steps, e.clip_grad_norm) == (0.01, "cosine", 100, 1.0)
    from bflc_demo_b200.ops.optim import OptimRecipe
    r = OptimRecipe.from_config(e)
    assert not r.is_default and r.schedule_id == 2 and OptimRecipe.from_config(c).is_default


@pytest.mark.parametrize("args", [["--weight-decay", "-1"], ["--lr-schedule", "step"], ["--warmup-steps", "-2"],
                                  ["--lr-schedule", "linear", "--warmup-steps", "4", "--total-steps", "4"],
                                  ["--clip-grad-norm", "-0.5"],
                                  ["--lr-schedule", "cosine", "--warmup-steps", "100000"]])
def test_run_rejects_bad_recipe_flags(args):
    from bflc_demo_b200.run import main
    with pytest.raises(SystemExit) as ei:
        main(["--model", "bert", *args])
    assert ei.value.code == 2


@pytest.mark.parametrize("args", [["--weight-decay", "0.01"], ["--clip-grad-norm", "1"], ["--warmup-steps", "2"],
                                  ["--lr-schedule", "linear"]])
def test_run_rejects_recipe_with_fused_mlp(args, capsys):
    from bflc_demo_b200.run import main
    with pytest.raises(SystemExit) as ei:
        main(["--model", "mlp", *args])
    assert ei.value.code == 2
    assert "--generic" in capsys.readouterr().err


@pytest.mark.parametrize("engine", ["fused", "nccl"])
def test_other_engines_reject_the_recipe(engine):
    cfg = FLConfig.for_world(1, clip_grad_norm=1.0)
    if engine == "fused":
        from bflc_demo_b200.engine.fused import FusedEngine as E
    else:
        from bflc_demo_b200.engine.nccl_baseline import NcclBaselineEngine as E
    with pytest.raises(ValueError, match="GenericFedEngine"):
        E(cfg, None)


def test_run_total_steps_default():
    import argparse
    from bflc_demo_b200.run import add_recipe_args, recipe_fields
    ap = argparse.ArgumentParser()
    add_recipe_args(ap)
    assert recipe_fields(ap, ap.parse_args(["--lr-schedule", "linear"]), 40)["total_steps"] == 40
    assert recipe_fields(ap, ap.parse_args([]), 40)["total_steps"] == 0     # constant: the defaults stay
    assert not FLConfig(**recipe_fields(ap, ap.parse_args([]), 40)).has_optim_recipe


# ------------------------------------------------------------------------- compiler guard
SRC = build.CSRC / "kernels" / "elementwise_optim.cu"
# registers of the plain instantiations (kAdam) before the recipe existed, sm_90a with build.py's flags
PLAIN_REGISTERS = {False: 31, True: 47}


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
    props = {}
    for name, st, ld, regs in re.findall(
            r"Function properties for \w*?\d(k_optimILb[01]ELb[01]E|k_grad_norm)\w*\s*\n\s*"
            r"\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\s*\n"
            r"ptxas info\s*: Used (\d+) registers", log):
        props[name] = (int(st), int(ld), int(regs))
    return props, log


def test_recipe_kernels_present_and_spill_free(ptxas_props):
    props, log = ptxas_props
    for name in ("k_optimILb0ELb1E", "k_optimILb1ELb1E", "k_grad_norm"):
        assert name in props, log[-3000:]
        st, ld, _ = props[name]
        assert st == 0 and ld == 0, f"{name}: {st} B spill stores / {ld} B loads"


def test_plain_optimizer_register_counts(ptxas_props):
    props, _ = ptxas_props
    for adam, want in PLAIN_REGISTERS.items():
        name = f"k_optimILb{int(adam)}ELb0E"
        st, ld, regs = props[name]
        assert (st, ld, regs) == (0, 0, want), name
