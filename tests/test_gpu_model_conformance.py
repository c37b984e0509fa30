"""Model conformance: LeNet-5, ResNet-18, BERT and the MLP through ``ops.nn`` against fp64, stage by
stage and end to end, on the flat parameter buffers the generic engine trains.

A recorder (``Recorder``) monkeypatches the layer functions ``models/nets.py`` calls through the
``ops.nn`` module object.  Each wrapper resolves every parameter argument to its ``ParamSpec`` entry
(by ``data_ptr`` inside the bound master / shadow / grad buffers), records the hyper-parameters and
clones of the op's inputs and output, and wraps the activation inputs and the output in an identity
autograd Function (``Tap``) that records the gradient passing through it and hands it on unchanged,
so each op's own ``dx`` and its upstream ``dy`` are captured without changing what the kernels do.

Checks, per case (``check_case``; each failure names its check):
* sequence -- the recorded calls equal an expected call list written here from the documented
  architectures (the class docstrings and BASELINE.json): op, parameter entries, hyper-parameters;
  every spec entry is used by exactly one call (``test_expected_calls_cover_the_spec``, CPU).
* edges -- each activation input is bit for bit the output of the call the list names (reshapes
  allowed); where a tensor feeds several consumers, its ``dy`` is the fp64 sum of their ``dx``
  within the (n - 1) bf16 roundings of autograd's accumulation, and exactly it for one consumer.
* stage -- every call against fp64 of that single op from its own recorded operands and ``dy``
  (ReLU masks from the kernel's own output), with elementwise bounds built from the fp32
  accumulation depth, the bf16 storage points and the imported layer / attention bounds.
* flat -- after one backward from a zeroed grad buffer: the grad gaps between entries and the tail,
  the padding slices of LeNet and the ResNet stem, every running-stat grad slot, the word rows of
  ids not in the batch and the position rows past the longest position are exactly zero; the
  master is unchanged by the forward except for the running statistics.
* e2e -- the loss, every gradient view and the running statistics against an independent fp64
  model written here (``fp64_forward``), norm-wise per view:
  ``||kernel - fp64|| <= 2 ||emulation - fp64|| + floor``, the emulation being the same model with
  a bf16 rounding at every point the kernels store bf16 (attention as the kernels compute it:
  ``AttnEmu``).  The loss gets a floor of half a bf16 ulp of itself, every other view 2^-16 of its
  norm; views that are zero in exact arithmetic (the key biases) and class-bias views of a few
  elements are reported, not held to the ratio.  The observed ratios are printed.
* hits -- the head's hit count in training and ``FlatNet.correct`` inside the fp64 range of
  ``test_gpu_val_split._fp64_hit_range``'s kind.

``test_checker_reports_mistake`` injects eight modelled mistakes at Python level and asserts the
checker reports each one and which check fired.  The ``LinearXentFn`` tests pin the head's
autograd contract: gradients scale with the upstream gradient, and a forward that is never
backpropagated leaves the gradient buffer alone.
"""
from __future__ import annotations

import inspect
import math
import sys
import time
import zlib
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as TF
from torch.autograd import Function

from bflc_demo_b200.models import nets
from bflc_demo_b200.ops import gemm as G
from bflc_demo_b200.ops import nn as NN

sys.path.insert(0, str(Path(__file__).resolve().parent))
from test_dropout_host import attention_keep_ref, hidden_keep_ref  # noqa: E402
from test_gpu_attention_conformance import bwd_bounds, fwd_bounds, ref_bwd, ref_fwd  # noqa: E402
from test_gpu_attention_conformance import violations as attn_violations  # noqa: E402
from test_gpu_gemm_conformance import acc_bound  # noqa: E402
from test_gpu_layer_conformance import (bn_stats_ref, bound_violations, colsum_ref, conv_dw_ref,  # noqa: E402
                                        conv_dx_ref, conv_ref, gelu_ref, im2col_ref, ln_stats_ref,
                                        maxpool_ref)

gpu = pytest.mark.gpu
BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24          # one fp32 rounding
BFU = 2.0 ** -8         # half a bf16 ulp, relative
TINY = 2.0 ** -120
GELU2 = 0.8             # max |gelu''| = 2 phi(0) < 0.8
GELU1 = 1.13            # max |gelu'|
SEED, STEP, ADD = 0x5EED_0123_4567_89AB, 3, 1
RATIO = 2.0             # e2e: ||kernel - fp64|| <= RATIO ||emulation - fp64|| + floor


class Mismatch(AssertionError):
    def __init__(self, check, msg):
        super().__init__(f"[{check}] {msg}")
        self.check = check


def fail(check, msg):
    raise Mismatch(check, msg)


def gam(n):
    """Worst-case relative error of an fp32 sum of n terms in any order (one ulp per addition)."""
    return 2 * n * U / (1 - 2 * n * U)


# ------------------------------------------------------------------------------- the recorder
class Tap(Function):
    """Identity; records the gradient flowing through it and returns it unchanged."""

    @staticmethod
    def forward(ctx, x, slot, key):
        ctx.set_materialize_grads(False)
        ctx.slot, ctx.key = slot, key
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        ctx.slot[ctx.key] = None if g is None else g.detach().clone()
        return g, None, None


ACTS = {"linear": ("x",), "linear_xent": ("h",), "conv2d": ("x",), "batchnorm": ("x", "residual"),
        "maxpool2d": ("x",), "global_avgpool": ("x",), "add": ("a", "b"), "layernorm": ("x",),
        "embedding": (), "attention": ("q", "k", "v"), "attention_packed": ("q", "k", "v"),
        "dropout_add": ("x", "z"), "dropout": ("z",)}
PARAMS = ("w", "b", "gw", "gb", "gamma", "beta", "ggamma", "gbeta", "run_mean", "run_var", "table", "pos",
          "gtable", "gpos")


class Recorder:
    """Context manager: records every ``ops.nn`` call a model makes (see the module docstring)."""

    def __init__(self, monkeypatch, spec, bufs):
        self.mp, self.spec, self.bufs = monkeypatch, spec, bufs
        self.calls, self.depth, self.lse = [], 0, []

    def name(self, t):
        if t is None:
            return None
        p = t.data_ptr()
        for tag, flat in self.bufs.items():
            es = flat.element_size()
            base = flat.data_ptr()
            if base <= p < base + flat.numel() * es and t.dtype == flat.dtype:
                off = (p - base) // es
                for e in self.spec.entries:
                    if e.offset <= off < e.offset + e.numel:
                        whole = off == e.offset and t.numel() == e.numel
                        return f"{tag}:{e.name}" + ("" if whole else f"[{off - e.offset}+{t.numel()}]")
                return f"{tag}:gap@{off}"
        return "foreign"

    def _wrap(self, op, fn):
        sig = inspect.signature(fn)
        rec_self = self

        def wrapper(*args, **kw):
            if rec_self.depth:
                return fn(*args, **kw)
            ba = sig.bind(*args, **kw)
            ba.apply_defaults()
            a = dict(ba.arguments)
            r = {"op": op, "params": {}, "hp": {}, "in": {}, "dx": {}, "dy": None}
            for k, v in a.items():
                if k in ACTS[op]:
                    if v is None:
                        r["hp"][k + "_given"] = False
                        continue
                    if op in ("batchnorm",) and k == "residual":
                        r["hp"]["residual_given"] = True
                    r["in"][k] = v.detach().clone()
                    if torch.is_grad_enabled() and v.requires_grad:
                        a[k] = Tap.apply(v, r["dx"], k)
                elif k in PARAMS:
                    r["params"][k] = rec_self.name(v)
                elif isinstance(v, NN.DropoutRNG):
                    r["hp"][k] = (int(v.seed), int(v.step[0]), int(v.add))
                elif torch.is_tensor(v):
                    r["hp"][k] = v.detach().clone()
                else:
                    r["hp"][k] = v
            if op == "batchnorm":
                r["run_before"] = (a["run_mean"].clone(), a["run_var"].clone())
                r["pv"] = {k: a[k].detach().double() for k in ("gamma", "beta")}
            if op == "layernorm":
                r["pv"] = {k: a[k].detach().double() for k in ("gamma", "beta")}
            if op in ("linear", "linear_xent", "conv2d"):
                r["pv"] = {"w": a["w"].detach().double(), "b": None if a["b"] is None else a["b"].detach().double()}
            if op == "embedding":
                r["pv"] = {"table": a["table"].detach().double(), "pos": a["pos"].detach().double()}
            n_lse = len(rec_self.lse)
            rec_self.depth += 1
            try:
                out = fn(**a)
            finally:
                rec_self.depth -= 1
            if op == "batchnorm":
                r["run_after"] = (a["run_mean"].clone(), a["run_var"].clone())
            if len(rec_self.lse) > n_lse:
                r["lse"] = rec_self.lse[-1]
            r["out"] = out.detach().clone()
            r["grad_mode"] = torch.is_grad_enabled()
            rec_self.calls.append(r)
            if torch.is_grad_enabled() and out.requires_grad:
                out = Tap.apply(out, r, "dy")
            return out

        return wrapper

    def __enter__(self):
        for op in ACTS:
            self.mp.setattr(NN, op, self._wrap(op, getattr(NN, op)))
        from bflc_demo_b200._native import C
        mod = C()
        for fname in ("attention_fwd", "attention_packed_fwd"):
            orig = getattr(mod, fname)

            def grab(*args, _orig=orig, **kw):
                res = _orig(*args, **kw)
                self.lse.append(args[4].clone())
                return res

            self.mp.setattr(mod, fname, grab)
        return self

    def __exit__(self, *exc):
        return False


# ---------------------------------------------------------------- the expected call lists
def E(cid, op, params=None, hp=None, ins=None):
    return {"id": cid, "op": op, "params": params or {}, "hp": hp or {}, "ins": ins or {}}


def lin(cid, src, act=G.ACT_NONE, need_dx=True):
    return E(cid, "linear", {"w": f"S:{cid}.w", "b": f"P:{cid}.b", "gw": f"G:{cid}.w", "gb": f"G:{cid}.b"},
             {"act": act, "need_dx": need_dx}, {"x": src})


def conv(cid, src, k, stride, pad, act=G.ACT_NONE, bias=True, need_dx=True):
    b = {"b": f"P:{cid}.b", "gb": f"G:{cid}.b"} if bias else {"b": None, "gb": None}
    return E(cid, "conv2d", {"w": f"S:{cid}.w", "gw": f"G:{cid}.w", **b},
             {"kh": k, "kw": k, "stride": stride, "pad": pad, "act": act, "need_dx": need_dx}, {"x": src})


def bn(cid, src, relu, res=None, training=True):
    ins = {"x": src}
    if res is not None:
        ins["residual"] = res
    return E(cid, "batchnorm", {"gamma": f"P:{cid}.gamma", "beta": f"P:{cid}.beta", "ggamma": f"G:{cid}.gamma",
                                "gbeta": f"G:{cid}.beta", "run_mean": f"P:{cid}.rmean", "run_var": f"P:{cid}.rvar"},
             {"training": training, "relu": relu, "residual_given": res is not None}, ins)


def ln(cid, src):
    return E(cid, "layernorm", {"gamma": f"P:{cid}.gamma", "beta": f"P:{cid}.beta", "ggamma": f"G:{cid}.gamma",
                                "gbeta": f"G:{cid}.beta"}, {}, {"x": src})


def head(w, src):
    return E("head", "linear_xent", {"w": f"S:{w}.w", "b": f"P:{w}.b", "gw": f"G:{w}.w", "gb": f"G:{w}.b"}, {},
             {"h": src})


def expected_mlp():
    return [lin("fc1", "input", G.ACT_RELU, need_dx=False), head("fc", "fc1")]


def expected_lenet():
    return [conv("conv1", "input", 5, 1, 0, G.ACT_RELU, need_dx=False),
            E("pool1", "maxpool2d", hp={"k": 2, "stride": 2, "pad": 0}, ins={"x": "conv1"}),
            conv("conv2", "pool1", 5, 1, 0, G.ACT_RELU),
            E("pool2", "maxpool2d", hp={"k": 2, "stride": 2, "pad": 0}, ins={"x": "conv2"}),
            lin("fc1", "pool2", G.ACT_RELU), lin("fc2", "fc1", G.ACT_RELU), head("fc", "fc2")]


def expected_resnet(widths=(64, 128, 256, 512), train=True):
    """CIFAR ResNet-18: 3x3 stem (no bias) + BN-ReLU, four stages of two BasicBlocks (3x3 conv
    stride s, BN-ReLU, 3x3 conv, BN + shortcut, ReLU; the shortcut a 1x1 strided conv + BN where the
    shape changes), global average pool, fc."""
    out = [conv("stem", "input", 3, 1, 1, bias=False, need_dx=False), bn("stem.bn", "stem", True, training=train)]
    x, cin = "stem.bn", widths[0]
    for si, c in enumerate(widths):
        for bi in range(2):
            n = f"l{si}.{bi}"
            s = 2 if si > 0 and bi == 0 else 1
            out += [conv(f"{n}.c1", x, 3, s, 1, bias=False), bn(f"{n}.bn1", f"{n}.c1", True, training=train),
                    conv(f"{n}.c2", f"{n}.bn1", 3, 1, 1, bias=False)]
            res = x
            if s != 1 or cin != c:
                out += [conv(f"{n}.down", x, 1, s, 0, bias=False), bn(f"{n}.dbn", f"{n}.down", False, training=train)]
                res = f"{n}.dbn"
            out.append(bn(f"{n}.bn2", f"{n}.c2", True, res, training=train))
            x, cin = f"{n}.bn2", c
    return out + [E("gap", "global_avgpool", ins={"x": x}), head("fc", "gap")]


def expected_bert(L, mode, p, lengths, B, S, H):
    """Post-LN BERT encoder: embedding + LN (+ dropout), per layer q/k/v, attention, o, residual
    (+ dropout), LN, GELU FFN, residual (+ dropout), LN; GELU pooler on [CLS] (+ dropout); head.
    ``mode``: "padded" (lengths None: unmasked) or "packed"."""
    site = nets.BertBase.dropout_site
    packed = mode == "packed"
    rows = {"S": None} if packed else {"S": S}
    out = [E("emb", "embedding", {"table": "S:emb.word", "pos": "S:emb.pos", "gtable": "G:emb.word",
                                  "gpos": "G:emb.pos"}, {"seq": 512 if packed else S}), ln("emb.ln", "emb")]
    x = "emb.ln"
    if p > 0:
        out.append(E("emb.drop", "dropout", hp={"p": p, "site": site(0, 0), **rows}, ins={"z": x}))
        x = "emb.drop"
    for i in range(L):
        e = f"enc{i}"
        out += [lin(f"{e}.q", x), lin(f"{e}.k", x), lin(f"{e}.v", x)]
        qkv = {"q": f"{e}.q", "k": f"{e}.k", "v": f"{e}.v"}
        if packed:
            out.append(E(f"{e}.attn", "attention_packed", hp={"H": H, "dropout_p": p, "site": site(i, 1)}, ins=qkv))
        else:
            out.append(E(f"{e}.attn", "attention", hp={"B": B, "S": S, "H": H, "fused": True, "dropout_p": p,
                                                        "site": site(i, 1)}, ins=qkv))
        out.append(lin(f"{e}.o", f"{e}.attn"))

        def res(cid, a, z, kind):
            if p > 0:
                return E(cid, "dropout_add", hp={"p": p, "site": site(i, kind), **rows}, ins={"x": a, "z": z})
            return E(cid, "add", ins={"a": a, "b": z})

        out += [res(f"{e}.res1", x, f"{e}.o", 2), ln(f"{e}.ln1", f"{e}.res1"),
                lin(f"{e}.ff1", f"{e}.ln1", G.ACT_GELU), lin(f"{e}.ff2", f"{e}.ff1"),
                res(f"{e}.res2", f"{e}.ln1", f"{e}.ff2", 3), ln(f"{e}.ln2", f"{e}.res2")]
        x = f"{e}.ln2"
    out.append(lin("pool", (x, "cls"), G.ACT_GELU))
    x = "pool"
    if p > 0:
        out.append(E("pool.drop", "dropout", hp={"p": p, "site": site(0, 4), "S": 1, "seq_ids": None,
                                                 "pos_ids": None}, ins={"z": x}))
        x = "pool.drop"
    return out + [head("cls", x)]


def spec_names_used(expected):
    used = {}
    for e in expected:
        for v in e["params"].values():
            if v is not None:
                nm = v.split(":", 1)[1]
                used.setdefault(nm, set()).add(e["id"])
    return used


# --------------------------------------------------------------------------------- cases
class Case:
    def __init__(self, cid, family, B, **kw):
        self.id, self.family, self.B, self.kw = cid, family, B, kw

    def __repr__(self):
        return self.id


CASES = [
    Case("mlp-b200", "mlp", 200),
    Case("lenet-b64", "lenet", 64),
    Case("lenet-b37", "lenet", 37),
    Case("resnet-b4", "resnet", 4),
    Case("bert-s128", "bert", 4, S=128),
    Case("bert-padded", "bert", 5, S=128, pad=True),
    Case("bert-packed", "bert", 5, S=128, pad=True, packed=True),
    Case("bert-drop-padded", "bert", 4, S=128, pad=True, p=0.1),
    Case("bert-drop-packed", "bert", 4, S=128, pad=True, packed=True, p=0.1),
    Case("bert-s96", "bert", 3, S=96),
    Case("mlp-mx8", "mlp", 200, mx8=True),
    Case("lenet-mx8", "lenet", 64, mx8=True),
]
BERT_LENS = {5: [128, 1, 77, 64, 100], 4: [1, 128, 65, 90]}


def make_net(c):
    if c.family == "mlp":
        return nets.MLPNet(784, 256, 62)
    if c.family == "lenet":
        return nets.LeNet5(10)
    if c.family == "resnet":
        return nets.ResNet18(10)
    return nets.BertBase(2, layers=2, pad_id=0 if c.kw.get("pad") else None, packed=c.kw.get("packed", False),
                         dropout=c.kw.get("p", 0.0))


def bert_lengths(c):
    return BERT_LENS[c.B] if c.kw.get("pad") else None


def expected_for(c, net):
    if c.family == "mlp":
        return expected_mlp()
    if c.family == "lenet":
        return expected_lenet()
    if c.family == "resnet":
        return expected_resnet(net.widths)
    return expected_bert(net.L, "packed" if net.packed else "padded", net.dropout, bert_lengths(c), c.B,
                         c.kw["S"], net.heads)


def make_data(c, net, dev="cuda"):
    g = torch.Generator().manual_seed(zlib.crc32(c.id.encode()))
    if c.family == "mlp":
        xr = torch.randint(0, 256, (c.B, 784), generator=g, dtype=torch.uint8)
    elif c.family in ("lenet", "resnet"):
        xr = torch.randint(0, 256, (c.B, 3, 32, 32), generator=g, dtype=torch.uint8)
    else:
        S = c.kw["S"]
        xr = torch.randint(1, 30522, (c.B, S), generator=g)
        lens = bert_lengths(c)
        if lens is not None:
            for b, n in enumerate(lens):
                xr[b, n:] = 0
    y = torch.randint(0, net.n_classes, (c.B,), generator=g, dtype=torch.int32)
    return xr.to(dev), y.to(dev)


def make_buffers(net, seed=1):
    master = torch.empty(net.spec.total)
    net.init_(master, seed=seed)
    if isinstance(net, nets.ResNet18):   # non-trivial running statistics and norm parameters
        g = torch.Generator().manual_seed(seed + 7)
        for k, v in net.spec.views(master).items():
            if k.endswith(".rmean"):
                v.copy_(torch.randn(v.shape, generator=g) * 0.1)
            elif k.endswith(".rvar"):
                v.copy_(torch.rand(v.shape, generator=g) + 0.5)
            elif k.endswith(".gamma"):
                v.copy_(torch.rand(v.shape, generator=g) + 0.5)
            elif k.endswith(".beta"):
                v.copy_(torch.randn(v.shape, generator=g) * 0.1)
    if isinstance(net, nets.BertBase):
        g = torch.Generator().manual_seed(seed + 9)
        for k, v in net.spec.views(master).items():
            if k.endswith(".b") or k.endswith(".beta"):
                v.copy_(torch.randn(v.shape, generator=g) * 0.02)
            elif k.endswith(".gamma"):
                v.copy_(1 + torch.randn(v.shape, generator=g) * 0.05)
    return master


# ------------------------------------------------------------------------ the kernel run
def run_kernels(c, monkeypatch, mutate=None):
    """One training forward + backward (and ``FlatNet.correct``) under the recorder."""
    net = make_net(c)
    master = make_buffers(net).cuda()
    shadow = master.to(BF16)
    grad = torch.zeros_like(master)
    xr, y = make_data(c, net)
    x = net.preprocess(xr)
    if mutate is not None:
        mutate(monkeypatch)
    prev = NN.set_precision("mx8" if c.kw.get("mx8") else "bf16")
    try:
        m0 = master.clone()
        b = net.bind(master, shadow, grad)
        rng = None
        if net.__class__ is nets.BertBase and net.dropout > 0:
            rng = NN.DropoutRNG(SEED, torch.tensor([STEP], device="cuda", dtype=torch.int32), ADD)
        cnt = torch.zeros(1, device="cuda", dtype=torch.int32)
        with Recorder(monkeypatch, net.spec, {"P": master, "S": shadow, "G": grad}) as rec:
            loss = net.loss(b, x, y, correct=cnt, rng=rng)
            m1 = master.clone()
            loss.backward()
            n_train = len(rec.calls)
            hits_eval = net.correct(net.bind(master, shadow), x, y)
        torch.cuda.synchronize()
    finally:
        NN.set_precision(prev)
    return dict(net=net, master0=m0, master1=m1, master=master, shadow=shadow, grad=grad, x=x, xr=xr, y=y,
                loss=loss.detach(), calls=rec.calls[:n_train], eval_calls=rec.calls[n_train:], hits=int(cnt),
                hits_eval=int(hits_eval), rng=rng)


# ------------------------------------------------------------------------ sequence / edges
def _same(a, b):
    if torch.is_tensor(a) or torch.is_tensor(b):
        return torch.is_tensor(a) and torch.is_tensor(b) and a.shape == b.shape and torch.equal(a, b)
    return a == b


def check_sequence(run, expected, c):
    calls = run["calls"]
    ops_r = [r["op"] for r in calls]
    ops_e = [e["op"] for e in expected]
    if ops_r != ops_e:
        fail("sequence", f"ops {ops_r} != expected {ops_e}")
    net = run["net"]
    hp_extra = expected_tensor_hp(run, c)
    for r, e in zip(calls, expected):
        r["id"] = e["id"]
        for k, v in e["params"].items():
            if r["params"].get(k) != v:
                fail("sequence", f"{e['id']}: parameter {k} is {r['params'].get(k)}, expected {v}")
        want = dict(e["hp"])
        for k, v in hp_extra.get(e["op"], {}).items():
            want.setdefault(k, v)
        for k, v in want.items():
            if k not in r["hp"]:
                fail("sequence", f"{e['id']}: no hyper-parameter {k}")
            if not _same(r["hp"][k], v):
                fail("sequence", f"{e['id']}: {k} = {r['hp'][k]!r}, expected {v!r}")
    used = spec_names_used(expected)
    for ent in net.spec.entries:
        if len(used.get(ent.name, ())) != 1:
            fail("sequence", f"spec entry {ent.name} used by {sorted(used.get(ent.name, ()))}")


def expected_tensor_hp(run, c):
    """Hyper-parameters that are tensors, derived here from the raw ids, not from the model."""
    net = run["net"]
    if not isinstance(net, nets.BertBase):
        return {"linear_xent": {"labels": run["y"]}}
    lens = bert_lengths(c)
    out = {"linear_xent": {"labels": run["y"]}}
    rng = (SEED, STEP, ADD) if net.dropout > 0 else None
    if net.packed:
        seq, pos = packed_coords(lens)
        cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device="cuda")
        out["embedding"] = {"pos_ids": pos}
        out["attention_packed"] = {"cu_seqlens": cu, "max_seqlen": max(lens)}
        if rng:
            out["attention_packed"]["rng"] = rng
            out["dropout"] = out["dropout_add"] = {"seq_ids": seq, "pos_ids": pos, "rng": rng}
    else:
        ln_t = None if lens is None else torch.tensor(lens, dtype=torch.int32, device="cuda")
        out["embedding"] = {"pos_ids": None}
        out["attention"] = {"lengths": ln_t}
        if rng:
            out["attention"]["rng"] = rng
            out["dropout"] = out["dropout_add"] = {"rng": rng}
    return out


def packed_coords(lens):
    seq = torch.tensor(np.repeat(np.arange(len(lens)), lens), dtype=torch.int32, device="cuda")
    pos = torch.tensor(np.concatenate([np.arange(n) for n in lens]), dtype=torch.int32, device="cuda")
    return seq, pos


def _source(run, src, c):
    """(tensor the edge should carry, producer id, transform)."""
    by_id = {r["id"]: r for r in run["calls"]}
    if src == "input":
        return run["x"], None, None
    if isinstance(src, tuple):
        pid, tr = src
        t = by_id[pid]["out"]
        net = run["net"]
        if net.packed:
            idx = torch.tensor(np.concatenate([[0], np.cumsum(bert_lengths(c))[:-1]]), device="cuda")
        else:
            idx = torch.arange(c.B, device="cuda") * c.kw["S"]
        return t.index_select(0, idx), pid, idx
    return by_id[src]["out"], src, None


def check_edges(run, expected, c):
    consumers = {}
    by_id = {r["id"]: r for r in run["calls"]}
    for e in expected:
        r = by_id[e["id"]]
        for name, src in e["ins"].items():
            want, pid, idx = _source(run, src, c)
            got = r["in"].get(name)
            if got is None or got.numel() != want.numel() or not torch.equal(got.reshape(-1), want.reshape(-1)):
                fail("edges", f"{e['id']}.{name} is not the output of {src}")
            if pid is not None:
                consumers.setdefault(pid, []).append((r, name, idx))
    for pid, cons in consumers.items():
        dy = by_id[pid]["dy"]
        parts = []
        for r, name, idx in cons:
            dx = r["dx"].get(name)
            if dx is None:
                continue
            dx = dx.double().reshape(-1, dx.shape[-1]) if idx is not None else dx.double()
            if idx is not None:
                full = torch.zeros(by_id[pid]["out"].shape, dtype=F64, device="cuda")
                full.index_copy_(0, idx, dx)
                dx = full
            parts.append(dx.reshape(by_id[pid]["out"].shape))
        if not parts:
            continue
        if dy is None:
            fail("edges", f"{pid}: consumers send gradient but none arrives")
        s = sum(parts)
        if len(parts) == 1:
            if not torch.equal(dy.double().reshape(s.shape), s):
                fail("edges", f"{pid}: dy differs from its one consumer's dx")
        else:
            tol = (len(parts) - 1) * BFU * sum(p.abs() for p in parts) * (1 + 2.0 ** -6) + TINY
            bad = (dy.double().reshape(s.shape) - s).abs() > tol
            if bool(bad.any()):
                fail("edges", f"{pid}: dy is not the sum of its {len(parts)} consumers' dx "
                              f"({int(bad.sum())} elements)")


# ------------------------------------------------------------------------- stage checks
def _assert(check, out, ref, slack, what):
    bad = bound_violations(out, ref, slack)
    if bool(bad.any()):
        i = tuple(int(j) for j in bad.nonzero()[0])
        fail(check, f"{what}: {int(bad.sum())} of {bad.numel()} wrong, first at {i}: "
                    f"{float(out[i])!r} vs {float(ref.to(out.device)[i])!r}")


def _exact(check, out, ref, what):
    if out.shape != ref.shape or not torch.equal(out.double(), ref.double()):
        fail(check, f"{what}: not exact")


def _mx(t):
    from bflc_demo_b200.ops.mx8 import quantize_mx8_reference
    return quantize_mx8_reference(t.float()).dequantize().double()


def act_fwd(z, ez, act, yk):
    """Reference output and slack of act(z) for a pre-activation z with error ez."""
    if act == G.ACT_RELU:
        return z.clamp(min=0), ez
    if act == G.ACT_GELU:
        return gelu_ref(z), GELU1 * ez + 8 * U * z.abs() + 2.0 ** -30
    return z, ez


def act_bwd(dy, z, ez, act, yk):
    """dz = dy * act'(z) with its slack; ReLU takes the kernel's own output as the mask."""
    dy = dy.double()
    if act == G.ACT_RELU:
        return dy * (yk.double() > 0), torch.zeros_like(dy)
    if act == G.ACT_GELU:
        g1 = 0.5 * (1 + torch.special.erf(z / 2 ** 0.5)) + z * torch.exp(-0.5 * z * z) / (2 * math.pi) ** 0.5
        dz = dy * g1
        e = dy.abs() * GELU2 * (ez + BFU * z.abs() + 2.0 ** -126) + 8 * U * dz.abs()
        return dz, e + BFU * (dz.abs() + e)
    return dy, torch.zeros_like(dy)


def grad_view(run, name):
    return run["net"].spec.views(run["grad"])[name]


def stage_gemm(run, r, A, quant, mm, mm_dx, mm_dw, K, rows, what, mx8=False):
    """Shared forward / backward check of linear and conv: ``mm(A, W)`` the fp64 product,
    ``mm_dx(dz, W)`` and ``mm_dw(A, dz)`` its transposes."""
    w, b = r["pv"]["w"], r["pv"]["b"]
    act = r["hp"]["act"]
    Af, wf = (A, w)
    if mx8:
        Af, wf = quant(A), quant(w)
    z = mm(Af, wf)
    ez = acc_bound(Af, wf, K)
    if b is not None:
        z = z + b
        ez = ez + 2 * U * b.abs()
    yk = r["out"].reshape(z.shape)
    yref, ey = act_fwd(z, ez, act, yk)
    _assert("stage", yk, yref, ey, f"{what} output")
    if r["dy"] is None:
        return
    dz, edz = act_bwd(r["dy"].reshape(z.shape), z, ez, act, yk)
    adz = dz.abs() + edz
    if r["params"]["gw"] is not None:
        gw = grad_view(run, r["params"]["gw"].split(":")[1]).reshape(w.shape)
        ref = mm_dw(A, dz)
        sl = mm_dw(A.abs(), edz) + gam(rows + 64) * mm_dw(A.abs(), adz)
        _assert("stage", gw, ref, sl, f"{what} weight gradient")
    if r["params"]["gb"] is not None:
        gb = grad_view(run, r["params"]["gb"].split(":")[1])
        red = dz.reshape(-1, dz.shape[-1])
        _assert("stage", gb, colsum_ref(red), colsum_ref(edz.reshape(red.shape))
                + gam(rows + 64) * colsum_ref(adz.reshape(red.shape)), f"{what} bias gradient")
    dx = r["dx"].get("x")
    if dx is not None:
        ref = mm_dx(dz, w)
        sl = mm_dx(edz, w.abs()) + gam(w.shape[0] * (K // max(1, w.shape[1])) + w.shape[0] + 64) * mm_dx(adz, w.abs())
        _assert("stage", dx, ref.reshape(dx.shape), sl.reshape(dx.shape), f"{what} dx")
    elif r["hp"]["need_dx"] and r["in"]["x"].requires_grad:
        fail("stage", f"{what}: no dx")


def stage_linear(run, r, mx8):
    x = r["in"]["x"].double()
    x2 = x.reshape(-1, x.shape[-1])
    stage_gemm(run, r, x2, _mx, lambda a, w: a @ w.t(), lambda dz, w: dz @ w, lambda a, dz: dz.t() @ a,
               x2.shape[1], x2.shape[0], r["id"], mx8=mx8 and r["hp"]["act"] != G.ACT_GELU)


def stage_conv(run, r, mx8):
    r["mx8"] = mx8
    x = r["in"]["x"].double()
    N, H, W, cin = x.shape
    k, s, p = r["hp"]["kh"], r["hp"]["stride"], r["hp"]["pad"]
    Kp = r["pv"]["w"].shape[1]
    w, b = r["pv"]["w"], r["pv"]["b"]
    OH, OW = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    if mx8:   # forward on the MXFP8-dequantised im2col operands (Kp columns); backward stays bf16
        col = torch.zeros(N * OH * OW, Kp, dtype=F64, device=x.device)
        col[:, :k * k * cin] = im2col_ref(x, k, s, p)
        cq, wq = _mx(col), _mx(w)
        z = (cq @ wq.t()).view(N, OH, OW, -1)
        ez = 2 * Kp * U * (cq.abs() @ wq.abs().t()).view(N, OH, OW, -1)
    else:
        z = conv_ref(x, w, k, s, p)
        ez = 2 * k * k * cin * U * conv_ref(x.abs(), w.abs(), k, s, p)
    if b is not None:
        z, ez = z + b, ez + 2 * U * b.abs()
    yk = r["out"].reshape(z.shape)
    yref, ey = act_fwd(z, ez, r["hp"]["act"], yk)
    _assert("stage", yk, yref, ey, f"{r['id']} output")
    stage_conv_bwd(run, r, x, z, ez)


def stage_conv_bwd(run, r, x, z, ez):
    if r["dy"] is None:
        return
    N, H, W, cin = x.shape
    k, s, p = r["hp"]["kh"], r["hp"]["stride"], r["hp"]["pad"]
    w = r["pv"]["w"]
    Kp, cout = w.shape[1], w.shape[0]
    yk = r["out"].reshape(z.shape)
    dz, edz = act_bwd(r["dy"].reshape(z.shape), z, ez, r["hp"]["act"], yk)
    adz = dz.abs() + edz
    rows = dz.numel() // cout
    gw = grad_view(run, r["params"]["gw"].split(":")[1])
    _assert("stage", gw, conv_dw_ref(x, dz, k, s, p, Kp),
            conv_dw_ref(x.abs(), edz, k, s, p, Kp) + gam(rows + 64) * conv_dw_ref(x.abs(), adz, k, s, p, Kp),
            f"{r['id']} weight gradient")
    if r["params"]["gb"] is not None:
        gb = grad_view(run, r["params"]["gb"].split(":")[1])
        _assert("stage", gb, colsum_ref(dz.reshape(-1, cout)),
                colsum_ref(edz.reshape(-1, cout)) + gam(rows + 64) * colsum_ref(adz.reshape(-1, cout)),
                f"{r['id']} bias gradient")
    dx = r["dx"].get("x")
    if dx is not None:
        ref = conv_dx_ref(dz, w, H, W, cin, k, s, p)
        sl = conv_dx_ref(edz, w.abs(), H, W, cin, k, s, p) \
            + gam(k * k * cout + 64) * conv_dx_ref(adz, w.abs(), H, W, cin, k, s, p)
        direct = (not r.get("mx8") and NN.conv_is_implicit(H, W, cin, k, k, s, p, Kp) and cout % 64 == 0
                  and NN._pix_tile(128, H, W))
        if not direct:   # dcol = dz @ w is stored in bf16 before col2im adds the taps up
            sl = sl + BFU * (1 + 2 * BFU) * conv_dx_ref(adz, w.abs(), H, W, cin, k, s, p)
        _assert("stage", dx, ref, sl, f"{r['id']} dx")


def stage_bn(run, r):
    x = r["in"]["x"].double()
    Cc = x.shape[-1]
    x2 = x.reshape(-1, Cc)
    rows = x2.shape[0]
    gamma, beta = r["pv"]["gamma"], r["pv"]["beta"]
    st = bn_stats_ref(x2)
    res = r["in"]["residual"].double().reshape(-1, Cc) if "residual" in r["in"] else None
    xc = x2 - st.mean
    xhat = xc * st.rstd
    exhat = st.mean_tol * st.rstd + xhat.abs() * (st.rstd_tol + 3 * U) + U * xc.abs() * st.rstd
    y = gamma * xhat + beta + (res if res is not None else 0)
    ey = gamma.abs() * exhat + 4 * U * (gamma.abs() * xhat.abs() + beta.abs() + (res.abs() if res is not None else 0))
    if r["hp"]["relu"]:
        y = y.clamp(min=0)
    yk = r["out"].reshape(-1, Cc)
    _assert("stage", yk, y, ey, f"{r['id']} output")
    rm0, rv0 = (t.double() for t in r["run_before"])
    rm1, rv1 = r["run_after"]
    rm_ref = 0.9 * rm0 + 0.1 * st.mean
    unb = rows / (rows - 1)
    rv_ref = 0.9 * rv0 + 0.1 * st.var * unb
    var_err = 2 * st.rstd_tol * (st.var + 1e-5)
    _assert("stage", rm1, rm_ref, 0.1 * st.mean_tol + 4 * U * (rm0.abs() + 0.1 * st.mean.abs()),
            f"{r['id']} running mean")
    _assert("stage", rv1, rv_ref, 0.1 * unb * var_err + 4 * U * (rv0.abs() + 0.1 * unb * st.var),
            f"{r['id']} running variance")
    if r["dy"] is None:
        return
    dy = r["dy"].double().reshape(-1, Cc)
    g = dy * (yk.double() > 0) if r["hp"]["relu"] else dy
    if res is not None:
        _exact("stage", r["dx"]["residual"].reshape(-1, Cc), g, f"{r['id']} residual gradient")
    n = rows + 64
    gb = grad_view(run, r["params"]["gbeta"].split(":")[1])
    gg = grad_view(run, r["params"]["ggamma"].split(":")[1])
    _assert("stage", gb, g.sum(0), gam(n) * g.abs().sum(0), f"{r['id']} beta gradient")
    _assert("stage", gg, (g * xhat).sum(0), (g.abs() * exhat).sum(0) + gam(n) * (g.abs() * xhat.abs()).sum(0),
            f"{r['id']} gamma gradient")
    mg, mgx = g.mean(0), (g * xhat).mean(0)
    core = g - mg - xhat * mgx
    e_mg = gam(n) * g.abs().mean(0)
    e_mgx = (g.abs() * exhat).mean(0) + gam(n) * (g * xhat).abs().mean(0)
    e_core = e_mg + exhat * mgx.abs() + xhat.abs() * e_mgx + exhat * e_mgx + 4 * U * (g.abs() + mg.abs() + (xhat * mgx).abs())
    dx = gamma * st.rstd * core
    edx = gamma.abs() * st.rstd * (e_core + core.abs() * (st.rstd_tol + 4 * U) + e_core * st.rstd_tol)
    _assert("stage", r["dx"]["x"].reshape(-1, Cc), dx, edx, f"{r['id']} dx")


def stage_ln(run, r):
    x = r["in"]["x"].double()
    rows, Cc = x.shape
    gamma, beta = r["pv"]["gamma"], r["pv"]["beta"]
    mean, rstd, mtol, rtol = ln_stats_ref(x)
    xc = x - mean[:, None]
    xhat = xc * rstd[:, None]
    exhat = mtol[:, None] * rstd[:, None] + xhat.abs() * (rtol[:, None] + 3 * U)
    y = gamma * xhat + beta
    ey = gamma.abs() * exhat + 4 * U * (gamma.abs() * xhat.abs() + beta.abs())
    _assert("stage", r["out"], y, ey, f"{r['id']} output")
    if r["dy"] is None:
        return
    dy = r["dy"].double()
    n = rows + 64
    gg = grad_view(run, r["params"]["ggamma"].split(":")[1])
    gb = grad_view(run, r["params"]["gbeta"].split(":")[1])
    _assert("stage", gb, dy.sum(0), gam(n) * dy.abs().sum(0), f"{r['id']} beta gradient")
    _assert("stage", gg, (dy * xhat).sum(0), (dy.abs() * exhat).sum(0) + gam(n) * (dy * xhat).abs().sum(0),
            f"{r['id']} gamma gradient")
    g = dy * gamma
    mg, mgx = g.mean(1, keepdim=True), (g * xhat).mean(1, keepdim=True)
    core = g - mg - xhat * mgx
    m = Cc + 64
    e_mg = gam(m) * g.abs().mean(1, keepdim=True) + 2 * U * g.abs().mean(1, keepdim=True)
    e_mgx = (g.abs() * exhat).mean(1, keepdim=True) + gam(m) * (g * xhat).abs().mean(1, keepdim=True)
    e_core = e_mg + exhat * mgx.abs() + xhat.abs() * e_mgx + exhat * e_mgx \
        + 4 * U * (g.abs() + mg.abs() + (xhat * mgx).abs())
    dx = rstd[:, None] * core
    edx = rstd[:, None] * (e_core * (1 + rtol[:, None]) + core.abs() * (rtol[:, None] + 4 * U))
    _assert("stage", r["dx"]["x"], dx, edx, f"{r['id']} dx")


def stage_embedding(run, r, c):
    ids = r["hp"]["ids"].long()
    table, pos = r["pv"]["table"], r["pv"]["pos"]
    net = run["net"]
    if net.packed:
        _, pid = packed_coords(bert_lengths(c))
        pid = pid.long()
    else:
        pid = torch.arange(ids.numel(), device="cuda") % c.kw["S"]
    ref = table[ids] + pos[pid]
    _assert("stage", r["out"], ref, U * ref.abs(), "embedding output")
    dy = r["dy"].double()
    gt, gp = grad_view(run, "emb.word"), grad_view(run, "emb.pos")
    ones = torch.ones(ids.numel(), 1, dtype=F64, device="cuda")
    for gv, idx, nm in ((gt, ids, "word"), (gp, pid, "position")):
        ref = torch.zeros(gv.shape, dtype=F64, device="cuda").index_add_(0, idx, dy)
        cnt = torch.zeros(gv.shape[0], 1, dtype=F64, device="cuda").index_add_(0, idx, ones)
        sl = gam(1) * cnt * torch.zeros(gv.shape, dtype=F64, device="cuda").index_add_(0, idx, dy.abs())
        _assert("stage", gv, ref, sl, f"embedding {nm} gradient")


def stage_maxpool(run, r):
    x = r["in"]["x"]
    k, s, p = r["hp"]["k"], r["hp"]["stride"], r["hp"]["pad"]
    y, idx = maxpool_ref(x, k, s, p)
    _exact("stage", r["out"].cpu(), y, f"{r['id']} output")
    if r["dy"] is None:
        return
    N, H, W, Cc = x.shape
    dx = torch.zeros(N, H * W * Cc, dtype=F64)
    d, i = r["dy"].double().cpu().reshape(N, -1), idx.reshape(N, -1)
    for n in range(N):
        dx[n].index_add_(0, i[n], d[n])
    _exact("stage", r["dx"]["x"].cpu(), dx.view(N, H, W, Cc).to(BF16), f"{r['id']} dx (first maximum)")


def stage_avgpool(run, r):
    x = r["in"]["x"].double()
    N, H, W, Cc = x.shape
    _assert("stage", r["out"], x.mean((1, 2)), gam(H * W + 8) * x.abs().mean((1, 2)), "avgpool output")
    dy = r["dy"].double()
    ref = (dy / (H * W))[:, None, None, :].expand(N, H, W, Cc)
    _assert("stage", r["dx"]["x"], ref, U * ref.abs(), "avgpool dx")


def stage_add(run, r):
    a, b = r["in"]["a"].double(), r["in"]["b"].double()
    _assert("stage", r["out"], a + b, U * (a + b).abs(), f"{r['id']} output")
    if r["dy"] is not None:
        for k in ("a", "b"):
            if r["dx"].get(k) is None or not torch.equal(r["dx"][k], r["dy"]):
                fail("stage", f"{r['id']}: gradient of operand {k} is not dy")


def _keep(r, c, rows, C):
    seed, step, add = r["hp"]["rng"]
    site, p = r["hp"]["site"], r["hp"]["p"]
    if r["hp"].get("seq_ids") is not None:
        seq, pos = r["hp"]["seq_ids"].cpu().numpy(), r["hp"]["pos_ids"].cpu().numpy()
    else:
        S = r["hp"]["S"]
        seq, pos = np.arange(rows) // S, np.arange(rows) % S
    keep = hidden_keep_ref(seed, step + add, site, p, seq, pos, C)
    ds = float(torch.tensor(1.0, dtype=F32) / (torch.tensor(1.0, dtype=F32) - torch.tensor(p, dtype=F32)))
    return torch.from_numpy(keep).to("cuda", F64) * ds


def stage_dropout(run, r, c):
    z = r["in"]["z"].double()
    rows, C = z.shape
    ks = _keep(r, c, rows, C)
    x = r["in"]["x"].double() if "x" in r["in"] else 0
    ref = x + z * ks
    _assert("stage", r["out"], ref, 2 * U * (z.abs() * ks + (x.abs() if torch.is_tensor(x) else 0)),
            f"{r['id']} output")
    if r["dy"] is None:
        return
    dy = r["dy"].double()
    _assert("stage", r["dx"]["z"], dy * ks, 2 * U * (dy * ks).abs(), f"{r['id']} dz (redrawn mask)")
    if "x" in r["in"] and not torch.equal(r["dx"]["x"], r["dy"]):
        fail("stage", f"{r['id']}: residual gradient is not dy")


def _heads(t, B, S, H):
    return t.double().reshape(B, S, H, 64).permute(0, 2, 1, 3).reshape(B * H, S, 64)


def stage_attention(run, r, c):
    hp = r["hp"]
    H = hp["H"]
    packed = r["op"] == "attention_packed"
    if packed:
        lens = bert_lengths(c)
        B, S = len(lens), (max(lens) + 63) // 64 * 64
        cu = np.concatenate([[0], np.cumsum(lens)])

        def lay(t):
            out = torch.zeros(B, S, H * 64, dtype=F64, device="cuda")
            for b in range(B):
                out[b, :lens[b]] = t[cu[b]:cu[b + 1]].double()
            return _heads(out, B, S, H)

        n = torch.tensor(lens, device="cuda")
    else:
        B, S = hp["B"], hp["S"]
        lay = lambda t: _heads(t, B, S, H)  # noqa: E731
        n = hp["lengths"].long().clamp(0, S) if hp["lengths"] is not None else torch.full((B,), S, device="cuda")
    kmask = (torch.arange(S, device="cuda")[None, :] < n[:, None]).repeat_interleave(H, 0)
    qmask = kmask if packed else torch.ones_like(kmask)
    if not packed and not NN.fused_attention_supported(S, 64):
        return stage_attention_unfused(r, B, S, H, lay)
    q, k, v = (lay(r["in"][x]) for x in ("q", "k", "v"))
    zs, ds = None, 1.0
    if hp["dropout_p"] > 0:
        seed, step, add = hp["rng"]
        ds = float(torch.tensor(1.0, dtype=F32) / (1 - torch.tensor(hp["dropout_p"], dtype=F32)))
        zs = torch.from_numpy(attention_keep_ref(seed, step + add, hp["site"], hp["dropout_p"], B, H, S)).to(
            "cuda", F64) * ds
    rowm = qmask[..., None]
    ok_ = lay(r["out"])
    rf = ref_fwd(q, k, v, kmask, 0.125, zs)
    fb = fwd_bounds(q, k, v, kmask, 0.125, rf, zs, ds)
    bad = attn_violations(ok_, rf["o"], fb["o"]) & rowm
    if bool(bad.any()):
        fail("stage", f"{r['id']} output: {int(bad.sum())} elements out of bound")
    if r["dy"] is None:
        return
    lse = r["lse"][:B * H * S].view(B * H, S).double()
    do = lay(r["dy"]) * rowm
    lse_in = torch.where(qmask, lse, 0.0)
    nq = 64 * torch.ceil(kmask.sum(-1).double() / 64)[:, None, None] if packed else float(S)
    rb = ref_bwd(q, k, v, do, ok_ * rowm, lse_in, kmask, 0.125, zs, qmask)
    bb = bwd_bounds(q, k, v, do, ok_ * rowm, lse_in, kmask, 0.125, rb, zs, ds, qmask, nq)
    for x in ("q", "k", "v"):
        bad = attn_violations(lay(r["dx"][x]), rb["d" + x], bb["d" + x]) & rowm
        if bool(bad.any()):
            fail("stage", f"{r['id']} d{x}: {int(bad.sum())} elements out of bound")


def stage_attention_unfused(r, B, S, H, lay):
    """``AttentionFn``: scores and probabilities are stored in bf16 between its GEMMs and the
    softmax kernel; the bound charges both roundings (and the fp32 sums) to each result."""
    q, k, v = (lay(r["in"][x]) for x in ("q", "k", "v"))
    sc = 0.125
    s = q @ k.mT
    es = gam(64) * (q.abs() @ k.abs().mT) + BFU * s.abs() * (1 + 2 * BFU)
    P = torch.softmax(sc * s, -1)
    rp = torch.exp(2 * sc * es.amax(-1, keepdim=True)) - 1 + 16 * U
    eP = P * rp + BFU * P * (1 + rp)
    o = P @ v
    eo = eP @ v.abs() + gam(S) * ((P + eP) @ v.abs())
    bad = attn_violations(lay(r["out"]), o, eo)
    if bool(bad.any()):
        fail("stage", f"{r['id']} output (unfused): {int(bad.sum())} out of bound")
    if r["dy"] is None:
        return
    do = lay(r["dy"])
    dP = do @ v.mT
    edP = gam(64) * (do.abs() @ v.abs().mT) + BFU * dP.abs() * (1 + 2 * BFU)
    delta = (P * dP).sum(-1, keepdim=True)
    edelta = (eP * dP.abs() + (P + eP) * edP).sum(-1, keepdim=True) + gam(S) * ((P + eP) * (dP.abs() + edP)).sum(-1, keepdim=True)
    A = dP - delta
    dS = P * A * sc
    edS = sc * (eP * A.abs() + (P + eP) * (edP + edelta) + 4 * U * (P + eP) * (A.abs() + edP + edelta))
    edS = edS + BFU * (dS.abs() + edS)
    aS = dS.abs() + edS
    want = {"q": (dS @ k, edS @ k.abs() + gam(S) * (aS @ k.abs())),
            "k": (dS.mT @ q, edS.mT @ q.abs() + gam(S) * (aS.mT @ q.abs())),
            "v": (P.mT @ do, eP.mT @ do.abs() + gam(S) * ((P + eP).mT @ do.abs()))}
    for x, (ref, sl) in want.items():
        bad = attn_violations(lay(r["dx"][x]), ref, sl)
        if bool(bad.any()):
            fail("stage", f"{r['id']} d{x} (unfused): {int(bad.sum())} out of bound")


def head_ref(h, w, b, y):
    """fp64 logits with their elementwise error bound (kernel fp32 sums + bias)."""
    z = h @ w.t() + b
    ez = gam(h.shape[1] + 1) * (h.abs() @ w.abs().t() + b.abs())
    return z, ez


def hit_range(h, w, b, y):
    z, ez = head_ref(h, w, b, y)
    top2 = z.topk(min(2, z.shape[1]), -1).values
    margin = top2[:, 0] - top2[:, 1]
    decided = margin > 2 * ez.amax(-1)
    hit = z.argmax(-1) == y.long()
    return int((hit & decided).sum()), int((~decided).sum())


def stage_head(run, r):
    h = r["in"]["h"].double()
    w, b = r["pv"]["w"], r["pv"]["b"]
    y = r["hp"]["labels"]
    M = h.shape[0]
    z, ez = head_ref(h, w, b, y)
    lse = torch.logsumexp(z, -1)
    lrow = lse - z.gather(1, y.long()[:, None])[:, 0]
    loss = lrow.mean()
    eloss = (2 * ez.amax(-1)).mean() + 16 * U * (lrow.abs() + lse.abs() + 1).mean() + gam(M) * lrow.abs().mean()
    if abs(float(r["out"].double().sum()) - float(loss)) > float(eloss) + BFU * 0 + 1e-30:
        fail("stage", f"head loss {float(r['out'].sum())!r} vs fp64 {float(loss)!r} (bound {float(eloss):.3g})")
    lo, und = hit_range(h, w, b, y)
    if not lo <= run["hits"] <= lo + und:
        fail("hits", f"training hits {run['hits']} outside [{lo}, {lo + und}]")
    P = torch.softmax(z, -1)
    dl = (P - TF.one_hot(y.long(), w.shape[0]).double()) / M
    mz = ez.amax(-1, keepdim=True)
    edl = (P * (torch.exp(2 * mz) - 1 + 8 * U) + 2 * U) / M
    edl = edl + BFU * (dl.abs() + edl)
    adl = dl.abs() + edl
    gw = grad_view(run, r["params"]["gw"].split(":")[1])
    gb = grad_view(run, r["params"]["gb"].split(":")[1])
    _assert("stage", gw, dl.t() @ h, edl.t() @ h.abs() + gam(M + 64) * (adl.t() @ h.abs()), "head weight gradient")
    _assert("stage", gb, dl.sum(0), edl.sum(0) + gam(M + 64) * adl.sum(0), "head bias gradient")
    if r["dx"].get("h") is not None:
        _assert("stage", r["dx"]["h"], dl @ w, edl @ w.abs() + gam(w.shape[0] + 8) * (adl @ w.abs()), "head dh")


def check_eval_hits(run):
    ev = run["eval_calls"]
    if not ev:
        fail("hits", "FlatNet.correct recorded no call")
    h = ev[-1]["out"].double()
    hd = run["net"].head
    V = run["net"].spec.views(run["shadow"])
    Pm = run["net"].spec.views(run["master"])
    lo, und = hit_range(h, V[hd[0]].double(), Pm[hd[1]].double(), run["y"])
    if not lo <= run["hits_eval"] <= lo + und:
        fail("hits", f"FlatNet.correct hits {run['hits_eval']} outside [{lo}, {lo + und}]")


def check_stages(run, c):
    mx8 = bool(c.kw.get("mx8"))
    for r in run["calls"]:
        op = r["op"]
        if op == "linear":
            stage_linear(run, r, mx8)
        elif op == "conv2d":
            stage_conv(run, r, mx8)
        elif op == "batchnorm":
            stage_bn(run, r)
        elif op == "layernorm":
            stage_ln(run, r)
        elif op == "embedding":
            stage_embedding(run, r, c)
        elif op == "maxpool2d":
            stage_maxpool(run, r)
        elif op == "global_avgpool":
            stage_avgpool(run, r)
        elif op == "add":
            stage_add(run, r)
        elif op in ("dropout", "dropout_add"):
            stage_dropout(run, r, c)
        elif op in ("attention", "attention_packed"):
            stage_attention(run, r, c)
        elif op == "linear_xent":
            stage_head(run, r)
    check_eval_hits(run)


# -------------------------------------------------------------------- flat-buffer invariants
def check_flat(run, c):
    net, grad = run["net"], run["grad"]
    spec = net.spec
    covered = torch.zeros(spec.total, dtype=torch.bool, device="cuda")
    for e in spec.entries:
        covered[e.offset:e.offset + e.numel] = True
    if bool(grad[:spec.total][~covered].any()):
        fail("flat", "gradient in the gaps between ParamSpec entries or the tail")
    Gv = spec.views(grad)
    zero = []
    if isinstance(net, nets.LeNet5):
        zero += [("conv1.w rows 6-7", Gv["conv1.w"][6:]), ("conv1.w columns 75-79", Gv["conv1.w"][:, 75:]),
                 ("conv2.w input channels 6-7", Gv["conv2.w"].view(16, 25, 8)[:, :, 6:]),
                 ("fc2.w rows 84-87", Gv["fc2.w"][84:]), ("fc.w columns 84-87", Gv["fc.w"][:, 84:])]
    if isinstance(net, nets.ResNet18):
        zero.append(("stem.w K pad", Gv["stem.w"][:, 27:]))
        zero += [(k, v) for k, v in Gv.items() if k.endswith(".rmean") or k.endswith(".rvar")]
    if isinstance(net, nets.BertBase):
        xr = run["xr"]
        lens = bert_lengths(c) or [c.kw["S"]] * c.B
        real = torch.cat([xr[b, :n] for b, n in enumerate(lens)]).long()
        used = torch.zeros(Gv["emb.word"].shape[0], dtype=torch.bool, device="cuda")
        used[real] = True
        zero += [("emb.word rows of ids not in the batch", Gv["emb.word"][~used]),
                 ("emb.pos rows past the longest position", Gv["emb.pos"][max(lens):])]
    for what, t in zero:
        if bool(t.any()):
            fail("flat", f"{what} not exactly zero")
    m0, m1 = run["master0"], run["master1"]
    moved = m0 != m1
    if isinstance(net, nets.ResNet18):
        for e in spec.entries:
            if e.name.endswith(".rmean") or e.name.endswith(".rvar"):
                moved[e.offset:e.offset + e.numel] = False
    if bool(moved.any()):
        fail("flat", "the forward changed the master outside the running statistics")


# -------------------------------------------------------------- independent fp64 models
class RoundBF(Function):
    """Emulation point: round the value (and the gradient passing back) to bf16."""

    @staticmethod
    def forward(ctx, x, fwd, bwd):
        ctx.bwd = bwd
        return x.to(BF16).to(x.dtype) if fwd else x.clone()

    @staticmethod
    def backward(ctx, g):
        return (g.to(BF16).to(g.dtype) if ctx.bwd else g), None, None


class MxMM(Function):
    """x @ w^T on MXFP8-dequantised operands forward, bf16 operands backward."""

    @staticmethod
    def forward(ctx, x, w):
        ctx.save_for_backward(x, w)
        return _mx(x) @ _mx(w).t()

    @staticmethod
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        return g @ w, g.t() @ x


def _bf(t):
    return t.to(BF16).to(t.dtype)


class AttnEmu(Function):
    """Emulated attention core on q, k, v [B, H, S, D] fp64 with the kernels' storage points.
    Fused (csrc/kernels/attn_sm100.cu): P (times the keep mask) rounded to bf16 before P V; the
    backward takes delta = rowsum(dO O) from the stored bf16 O and rounds dS to bf16.  Unfused
    (``AttentionFn``): scores, probabilities and dP stored in bf16, delta = rowsum(P dP)."""

    @staticmethod
    def forward(ctx, q, k, v, kmask, zs, scale, fused):
        s = q @ k.transpose(-1, -2)
        if not fused:
            s = _bf(s)
        P = torch.softmax((s * scale).masked_fill(~kmask[:, None, None, :], -math.inf), -1)
        if not fused:
            P = _bf(P)
        W = P if zs is None else P * zs
        O = _bf(_bf(W) @ v)
        ctx.save_for_backward(q, k, v, P, O)
        ctx.zs, ctx.scale, ctx.fused = zs, scale, fused
        return O

    @staticmethod
    def backward(ctx, dO):
        q, k, v, P, O = ctx.saved_tensors
        zs = ctx.zs
        W = P if zs is None else P * zs
        dv = _bf(W).transpose(-1, -2) @ dO
        dP = dO @ v.transpose(-1, -2)
        if ctx.fused:
            Gd = dP if zs is None else dP * zs
            delta = (dO * O).sum(-1, keepdim=True)
        else:
            Gd = dP = _bf(dP)
            delta = (P * dP).sum(-1, keepdim=True)
        dS = _bf(P * (Gd - delta) * ctx.scale)
        return dS @ k, dS.transpose(-1, -2) @ q, dv, None, None, None, None


class Model64:
    """Rounding hooks of one fp64 model run: ``emul`` False is the plain fp64 model."""

    def __init__(self, emul, mx8=False):
        self.emul, self.mx8 = emul, mx8

    def r(self, t):          # a stored bf16 activation (and its stored gradient)
        return RoundBF.apply(t, True, True) if self.emul else t

    def rg(self, t):         # a stored bf16 gradient only (dz, dlogits)
        return RoundBF.apply(t, False, True) if self.emul else t

    def mm(self, x, w):
        return MxMM.apply(x, w) if self.mx8 else x @ w.t()

    def linear(self, x, w, b, act=G.ACT_NONE):
        z = self.mm(x, w) + b
        if act == G.ACT_RELU:
            return self.r(torch.relu(self.rg(z)))
        if act == G.ACT_GELU:
            return self.r(gelu_ref(self.r(z)))
        return self.r(z)

    def conv(self, x, w, b, k, s, p, act=G.ACT_NONE):
        """x NHWC; w [Cout, Kp] channels-last taps."""
        N, H, W, cin = x.shape
        cout = w.shape[0]
        if self.mx8:
            col = im2col_ref(x, k, s, p)
            col = torch.cat([col, col.new_zeros(col.shape[0], w.shape[1] - col.shape[1])], 1)
            z = MxMM.apply(col, w).view(N, (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1, cout)
        else:
            wt = w[:, :k * k * cin].reshape(cout, k, k, cin).permute(0, 3, 1, 2)
            z = TF.conv2d(x.permute(0, 3, 1, 2), wt, None, s, p).permute(0, 2, 3, 1)
        if b is not None:
            z = z + b
        if act == G.ACT_RELU:
            return self.r(torch.relu(self.rg(z)))
        return self.r(z)

    def head_loss(self, h, w, b, y):
        z = self.rg(h @ w.t() + b)
        return TF.cross_entropy(z, y.long())


def fp64_forward(c, net, Pd, x, y, m, lens=None, rng=None):
    """The network written from its documented architecture.  ``Pd``: name -> fp64 leaf (shadow
    values for GEMM weights and embeddings, master values for the rest).  -> (loss, extras)."""
    extras = {}
    if isinstance(net, nets.MLPNet):
        h = m.linear(x, Pd["fc1.w"], Pd["fc1.b"], G.ACT_RELU)
        return m.head_loss(h, Pd["fc.w"], Pd["fc.b"], y), extras
    if isinstance(net, nets.LeNet5):
        t = m.conv(x, Pd["conv1.w"], Pd["conv1.b"], 5, 1, 0, G.ACT_RELU)
        t = TF.max_pool2d(t.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
        t = m.conv(t, Pd["conv2.w"], Pd["conv2.b"], 5, 1, 0, G.ACT_RELU)
        t = TF.max_pool2d(t.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1).reshape(x.shape[0], -1)
        t = m.linear(t, Pd["fc1.w"], Pd["fc1.b"], G.ACT_RELU)
        t = m.linear(t, Pd["fc2.w"], Pd["fc2.b"], G.ACT_RELU)
        return m.head_loss(t, Pd["fc.w"], Pd["fc.b"], y), extras
    if isinstance(net, nets.ResNet18):
        def bnf(t, name, relu, res=None):
            rm, rv = Pd[f"{name}.rmean"].detach().clone(), Pd[f"{name}.rvar"].detach().clone()
            C_ = t.shape[-1]
            o = TF.batch_norm(t.reshape(-1, C_), rm, rv, Pd[f"{name}.gamma"], Pd[f"{name}.beta"], True, 0.1,
                              1e-5).view(t.shape)
            extras[f"{name}.rmean"], extras[f"{name}.rvar"] = rm, rv
            if res is not None:
                o = o + res
            return m.r(torch.relu(m.rg(o)) if relu else o)

        t = m.conv(x, Pd["stem.w"], None, 3, 1, 1)
        t = bnf(t, "stem.bn", True)
        for name, cin, cc, s, down in net.blocks:
            u = m.conv(t, Pd[f"{name}.c1.w"], None, 3, s, 1)
            u = bnf(u, f"{name}.bn1", True)
            u = m.conv(u, Pd[f"{name}.c2.w"], None, 3, 1, 1)
            idt = t
            if down:
                idt = bnf(m.conv(t, Pd[f"{name}.down.w"], None, 1, s, 0), f"{name}.dbn", False)
            t = bnf(u, f"{name}.bn2", True, idt)
        t = m.r(t.mean((1, 2)))
        return m.head_loss(t, Pd["fc.w"], Pd["fc.b"], y), extras
    # BERT
    ids = x
    B, S = ids.shape
    Hd, H = net.Hd, net.heads
    D = Hd // H
    p = net.dropout if rng is not None else 0.0
    site = nets.BertBase.dropout_site
    n = torch.tensor(lens if lens is not None else [S] * B, device=ids.device)
    kmask = torch.arange(S, device=ids.device)[None, :] < n[:, None]
    dsc = float(torch.tensor(1.0, dtype=F32) / (1 - torch.tensor(p, dtype=F32))) if p else 1.0
    seqs, poss = np.arange(B * S) // S, np.arange(B * S) % S

    def hdrop(t, st):
        if not p:
            return t
        keep = hidden_keep_ref(SEED, STEP + ADD, st, p, seqs[:t.shape[0]] if t.shape[0] == B * S else np.arange(B),
                               poss if t.shape[0] == B * S else np.zeros(B, dtype=np.int64), t.shape[1])
        return t * (torch.from_numpy(keep).to(t.device, t.dtype) * dsc)

    def lnf(t, name):
        return m.r(TF.layer_norm(t, (Hd,), Pd[f"{name}.gamma"], Pd[f"{name}.beta"], 1e-12))

    t = m.r(Pd["emb.word"][ids.reshape(-1).long()] + Pd["emb.pos"][torch.arange(S, device=ids.device).repeat(B)])
    t = lnf(t, "emb.ln")
    t = m.r(hdrop(t, site(0, 0)))
    for i in range(net.L):
        e = f"enc{i}"
        q, k, v = (m.linear(t, Pd[f"{e}.{nm}.w"], Pd[f"{e}.{nm}.b"]).view(B, S, H, D).transpose(1, 2)
                   for nm in ("q", "k", "v"))
        zs = None
        if p:
            keep = attention_keep_ref(SEED, STEP + ADD, site(i, 1), p, B, H, S)
            zs = torch.from_numpy(keep).to(q.device, q.dtype).view(B, H, S, S) * dsc
        if m.emul:
            a = AttnEmu.apply(q, k, v, kmask, zs, 1 / math.sqrt(D), NN.fused_attention_supported(S, D))
        else:
            s = (q @ k.transpose(-1, -2)) / math.sqrt(D)
            P = torch.softmax(s.masked_fill(~kmask[:, None, None, :], -math.inf), -1)
            a = (P if zs is None else P * zs) @ v
        a = m.r(a).transpose(1, 2).reshape(B * S, Hd)
        a = m.linear(a, Pd[f"{e}.o.w"], Pd[f"{e}.o.b"])
        t = lnf(m.r(t + hdrop(a, site(i, 2))), f"{e}.ln1")
        f = m.linear(t, Pd[f"{e}.ff1.w"], Pd[f"{e}.ff1.b"], G.ACT_GELU)
        f = m.linear(f, Pd[f"{e}.ff2.w"], Pd[f"{e}.ff2.b"])
        t = lnf(m.r(t + hdrop(f, site(i, 3))), f"{e}.ln2")
    cls = t.view(B, S, Hd)[:, 0]
    pooled = m.linear(cls, Pd["pool.w"], Pd["pool.b"], G.ACT_GELU)
    pooled = m.r(hdrop(pooled, site(0, 4)))
    return m.head_loss(pooled, Pd["cls.w"], Pd["cls.b"], y), extras


def fp64_params(net, master, shadow, dev):
    V, Pm = net.spec.views(shadow), net.spec.views(master)
    out = {}
    for e in net.spec.entries:
        src = V if (e.name.endswith(".w") or e.name.startswith("emb.word") or e.name.startswith("emb.pos")) else Pm
        out[e.name] = src[e.name].detach().to(dev, F64).clone().requires_grad_(True)
    return out


def fp64_run(c, net, master, shadow, xr, y, emul, dev="cuda"):
    Pd = fp64_params(net, master, shadow, dev)
    if isinstance(net, nets.BertBase):
        x = xr.to(dev)
    else:
        x = net.preprocess(xr).to(dev, F64) if dev == "cuda" else None
    mx8 = bool(c.kw.get("mx8")) if c is not None else False
    rng = True if (isinstance(net, nets.BertBase) and net.dropout > 0) else None
    loss, extras = fp64_forward(c, net, Pd, x, y.to(dev), Model64(emul, mx8), bert_lengths(c) if c else None, rng)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in Pd.items()}
    return loss.detach(), grads, extras


def check_e2e(run, c, report):
    net = run["net"]
    f64 = fp64_run(c, net, run["master0"], run["shadow"], run["xr"], run["y"], False)
    emu = fp64_run(c, net, run["master0"], run["shadow"], run["xr"], run["y"], True)
    Gv = net.spec.views(run["grad"])
    Pm = net.spec.views(run["master"])
    items = [("loss", run["loss"].double().reshape(()), f64[0], emu[0])]
    for e in net.spec.entries:
        if e.name.endswith(".rmean") or e.name.endswith(".rvar"):
            items.append((e.name + " (running)", Pm[e.name].double(), f64[2][e.name], emu[2][e.name]))
        else:
            items.append((e.name, Gv[e.name].double(), f64[1][e.name], emu[1][e.name]))
    worst, bad = 0.0, []
    for name, k, ref, em in items:
        ek = float((k - ref.reshape(k.shape)).norm())
        ee = float((em.reshape(k.shape) - ref.reshape(k.shape)).norm())
        rn = float(ref.norm())
        # the loss is one draw of the rounding error, so its ratio is not a statistic: it gets half
        # a bf16 ulp of itself; every other view gets 2^-16 of its norm (fp32 sums)
        floor = (BFU if k.numel() == 1 else 2.0 ** -16) * rn + 1e-30
        ratio = ek / ee if ee > 0 else (0.0 if ek == 0 else math.inf)
        # not held to the ratio, only reported (the stage checks bound them elementwise): views that
        # are zero in exact arithmetic (the key biases, pure rounding noise), and views of a few
        # elements other than the loss (class biases: a handful of draws, often a cancelling sum)
        noise = rn < ee or 1 < k.numel() < 64
        report.append((name, ratio, ek, ee, noise))
        if noise:
            continue
        if ek > RATIO * ee + floor:
            bad.append(f"{name}: ||kernel - fp64|| = {ek:.3g} > {RATIO} x ||emulation - fp64|| = {ee:.3g} "
                       f"+ floor {floor:.3g}")
        if ee > 0:
            worst = max(worst, ek / ee)
    if bad:
        fail("e2e", f"{len(bad)} views: " + "; ".join(bad))
    return worst


def check_case(c, monkeypatch, mutate=None, e2e=True):
    run = run_kernels(c, monkeypatch, mutate)
    expected = expected_for(c, run["net"])
    check_sequence(run, expected, c)
    check_edges(run, expected, c)
    check_stages(run, c)
    check_flat(run, c)
    report = []
    worst = check_e2e(run, c, report) if e2e else None
    return run, report, worst


# ================================================================================== tests
@pytest.mark.parametrize("family", ["mlp", "lenet", "resnet", "bert-padded", "bert-packed", "bert-drop"])
def test_expected_calls_cover_the_spec(family):
    """Every ParamSpec entry is named by exactly one expected call, every edge points to an earlier
    call, ids are unique (CPU)."""
    if family == "mlp":
        net, exp = nets.MLPNet(784, 256, 62), expected_mlp()
    elif family == "lenet":
        net, exp = nets.LeNet5(10), expected_lenet()
    elif family == "resnet":
        net = nets.ResNet18(10)
        exp = expected_resnet(net.widths)
    else:
        p = 0.1 if family == "bert-drop" else 0.0
        packed = family == "bert-packed"
        net = nets.BertBase(2, layers=2, pad_id=0, packed=packed, dropout=p)
        exp = expected_bert(2, "packed" if packed else "padded", p, [3, 5], 2, 8, 12)
    ids = [e["id"] for e in exp]
    assert len(set(ids)) == len(ids)
    seen = set()
    for e in exp:
        for src in e["ins"].values():
            s = src[0] if isinstance(src, tuple) else src
            assert s == "input" or s in seen, f"{e['id']} reads {s} before it exists"
        seen.add(e["id"])
    used = spec_names_used(exp)
    assert sorted(used) == sorted(x.name for x in net.spec.entries)
    assert all(len(v) == 1 for v in used.values()), {k: v for k, v in used.items() if len(v) != 1}


def test_fp64_resnet_matches_stock_torch():
    """The functional fp64 ResNet against a BasicBlock stack of stock torch layers (small widths)."""
    import torch.nn as tnn
    torch.manual_seed(0)
    net = nets.ResNet18(10, widths=(8, 16, 16, 32))
    master = make_buffers(net)
    shadow = master.to(BF16)
    Pd = fp64_params(net, master, shadow, "cpu")
    x = torch.randn(3, 32, 32, 3, dtype=F64)
    y = torch.randint(0, 10, (3,))
    loss, ex = fp64_forward(None, net, Pd, x, y, Model64(False))

    def conv(name, cin, cout, k, s, p):
        m = tnn.Conv2d(cin, cout, k, s, p, bias=False).double()
        m.weight.data.copy_(Pd[name][:, :k * k * cin].detach().view(cout, k, k, cin).permute(0, 3, 1, 2))
        return m

    def bnm(name, c):
        m = tnn.BatchNorm2d(c, eps=1e-5, momentum=0.1).double()
        m.weight.data.copy_(Pd[f"{name}.gamma"].detach())
        m.bias.data.copy_(Pd[f"{name}.beta"].detach())
        m.running_mean.copy_(Pd[f"{name}.rmean"].detach())
        m.running_var.copy_(Pd[f"{name}.rvar"].detach())
        return m

    class Block(tnn.Module):
        def __init__(self, name, cin, c, s, down):
            super().__init__()
            self.c1, self.b1 = conv(f"{name}.c1.w", cin, c, 3, s, 1), bnm(f"{name}.bn1", c)
            self.c2, self.b2 = conv(f"{name}.c2.w", c, c, 3, 1, 1), bnm(f"{name}.bn2", c)
            self.down = tnn.Sequential(conv(f"{name}.down.w", cin, c, 1, s, 0), bnm(f"{name}.dbn", c)) if down else None

        def forward(self, t):
            o = torch.relu(self.b1(self.c1(t)))
            o = self.b2(self.c2(o))
            return torch.relu(o + (self.down(t) if self.down is not None else t))

    stem = tnn.Sequential(conv("stem.w", 3, 8, 3, 1, 1), bnm("stem.bn", 8), tnn.ReLU())
    blocks = tnn.Sequential(*[Block(*b) for b in net.blocks])
    fc = tnn.Linear(32, 10).double()
    fc.weight.data.copy_(Pd["fc.w"].detach())
    fc.bias.data.copy_(Pd["fc.b"].detach())
    model = tnn.Sequential(stem, blocks, tnn.AdaptiveAvgPool2d(1), tnn.Flatten(), fc).train()
    ref = TF.cross_entropy(model(x.permute(0, 3, 1, 2)), y)
    assert torch.allclose(loss, ref, rtol=1e-12, atol=1e-12)
    loss.backward()
    ref.backward()
    assert torch.allclose(Pd["fc.w"].grad, fc.weight.grad, rtol=1e-10, atol=1e-12)
    w0 = blocks[0].c1.weight.grad.permute(0, 2, 3, 1).reshape(8, -1)
    assert torch.allclose(Pd["l0.0.c1.w"].grad, w0, rtol=1e-10, atol=1e-12)
    assert torch.allclose(ex["l1.0.dbn.rvar"], blocks[2].down[1].running_var, rtol=1e-12)
    assert torch.allclose(ex["stem.bn.rmean"], stem[1].running_mean, rtol=1e-12, atol=1e-14)


def test_fp64_bert_matches_stock_torch():
    """The functional fp64 BERT encoder against ``nn.TransformerEncoderLayer`` (post-LN, GELU,
    eps 1e-12) with its weights copied in, key padding masked (small dims, CPU)."""
    import torch.nn as tnn
    torch.manual_seed(1)
    net = nets.BertBase(2, layers=2, hidden=64, heads=2, ffn=128, vocab=50, max_pos=16, pad_id=0)
    master = make_buffers(net)
    shadow = master.to(BF16)
    Pd = fp64_params(net, master, shadow, "cpu")
    lens = [16, 5, 1]
    ids = torch.randint(1, 50, (3, 16))
    for b, n in enumerate(lens):
        ids[b, n:] = 0
    y = torch.randint(0, 2, (3,))
    loss, _ = fp64_forward(None, net, Pd, ids, y, Model64(False), lens)
    layers = []
    for i in range(2):
        e = f"enc{i}"
        m = tnn.TransformerEncoderLayer(64, 2, 128, dropout=0.0, activation="gelu", layer_norm_eps=1e-12,
                                        batch_first=True, norm_first=False).double()
        m.self_attn.in_proj_weight.data.copy_(torch.cat([Pd[f"{e}.{n}.w"].detach() for n in "qkv"]))
        m.self_attn.in_proj_bias.data.copy_(torch.cat([Pd[f"{e}.{n}.b"].detach() for n in "qkv"]))
        m.self_attn.out_proj.weight.data.copy_(Pd[f"{e}.o.w"].detach())
        m.self_attn.out_proj.bias.data.copy_(Pd[f"{e}.o.b"].detach())
        for a, b_ in (("linear1", "ff1"), ("linear2", "ff2")):
            getattr(m, a).weight.data.copy_(Pd[f"{e}.{b_}.w"].detach())
            getattr(m, a).bias.data.copy_(Pd[f"{e}.{b_}.b"].detach())
        for a, b_ in (("norm1", "ln1"), ("norm2", "ln2")):
            getattr(m, a).weight.data.copy_(Pd[f"{e}.{b_}.gamma"].detach())
            getattr(m, a).bias.data.copy_(Pd[f"{e}.{b_}.beta"].detach())
        layers.append(m.eval())
    t = Pd["emb.word"].detach()[ids] + Pd["emb.pos"].detach()[:16][None]
    t = TF.layer_norm(t, (64,), Pd["emb.ln.gamma"].detach(), Pd["emb.ln.beta"].detach(), 1e-12)
    pad = ids == 0
    for m in layers:
        m.train()   # the math path (no fused fast path); dropout is 0
        t = m(t, src_key_padding_mask=pad)
    pooled = TF.gelu(t[:, 0] @ Pd["pool.w"].detach().t() + Pd["pool.b"].detach())
    ref = TF.cross_entropy(pooled @ Pd["cls.w"].detach().t() + Pd["cls.b"].detach(), y)
    assert torch.allclose(loss.detach(), ref, rtol=1e-11, atol=1e-12), (float(loss), float(ref))


def test_emulation_differs_from_fp64_but_stays_close():
    """The bf16 emulation moves the loss and the gradients by bf16-sized amounts, not 0 and not more."""
    net = nets.MLPNet(784, 256, 62)
    master = make_buffers(net)
    shadow = master.to(BF16)
    g = torch.Generator().manual_seed(3)
    x = torch.rand(64, 784, generator=g, dtype=F64).to(BF16).double()
    y = torch.randint(0, 62, (64,), generator=g)
    outs = []
    for emul in (False, True):
        Pd = fp64_params(net, master, shadow, "cpu")
        loss, _ = fp64_forward(None, net, Pd, x, y, Model64(emul))
        loss.backward()
        outs.append((loss.detach(), Pd["fc1.w"].grad.clone()))
    dl = float((outs[0][0] - outs[1][0]).abs())
    dg = float((outs[0][1] - outs[1][1]).norm() / outs[0][1].norm())
    assert 0 < dl < 1e-2 and 0 < dg < 3e-2, (dl, dg)


@gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_model_conformance(case, monkeypatch):
    t0 = time.perf_counter()
    torch.manual_seed(0)
    run, report, worst = check_case(case, monkeypatch)
    held = [r for r in report if math.isfinite(r[1]) and not r[4]]
    top = sorted(held, key=lambda r: -r[1])[:3]
    ratios = np.array([r[1] for r in held if r[3] > 0])
    noise = [f"{r[0]} {r[1]:.2f}" for r in report if r[4]]   # reported, not held to the ratio
    print(f"\n[e2e] {case.id}: ||kernel-fp64|| / ||emul-fp64|| over {len(ratios)} views: median "
          f"{np.median(ratios):.3f}, max {worst:.3f} ({', '.join(f'{r[0]} {r[1]:.3f}' for r in top)}); "
          f"loss {report[0][1]:.3f}; reported only: {noise or 'none'}; {time.perf_counter() - t0:.1f} s")


# -------------------------------------------------------------------------- checker teeth
def _m_add_drops_b(mp):
    mp.setattr(NN.AddFn, "backward", staticmethod(lambda ctx, g: (g, torch.zeros_like(g))))


def _m_xent_scale(mp):
    orig = G.gemm_xent

    def bad(a, b, labels, **kw):
        kw["grad_scale"] = 1.0 / (a.shape[0] + 1)
        return orig(a, b, labels, **kw)

    mp.setattr(G, "gemm_xent", bad)


def _m_ln_swap(mp):
    orig = NN.layernorm
    mp.setattr(NN, "layernorm", lambda x, gamma, beta, ggamma=None, gbeta=None: orig(x, gamma, beta, gbeta, ggamma))


def _m_pos_plus_one(mp):
    orig = NN.embedding

    def bad(ids, table, pos, gtable, gpos, seq, pos_ids=None):
        return orig(ids, table, pos, gtable, gpos, seq, None if pos_ids is None else pos_ids + 1)

    mp.setattr(NN, "embedding", bad)


def _m_pool_relu(mp):
    def bad(self, b, cls_tok, p, rng):
        pooled = self._lin(b, "pool", cls_tok, G.ACT_RELU)
        return NN.dropout(pooled, p, rng, self.dropout_site(0, self.SITE_POOL), S=1) if p > 0.0 else pooled

    mp.setattr(nets.BertBase, "_pool", bad)


def _m_dropout_site(mp):
    orig = NN.DropoutAddFn.backward

    def bad(ctx, dy):
        p, rng, site, S, seq_ids, pos_ids = ctx.args
        ctx.args = (p, rng, site + 1, S, seq_ids, pos_ids)
        return orig(ctx, dy)

    mp.setattr(NN.DropoutAddFn, "backward", staticmethod(bad))


def _m_bn_eval(mp):
    orig = nets.ResNet18._bn

    def bad(self, b, name, x, train, relu, residual=None):
        return orig(self, b, name, x, train and name != "l1.0.bn1", relu, residual)

    mp.setattr(nets.ResNet18, "_bn", bad)


def _m_lengths_plus_one(mp):
    orig = NN.attention

    def bad(q, k, v, B, S, H, fused=True, lengths=None, dropout_p=0.0, rng=None, site=0):
        return orig(q, k, v, B, S, H, fused, None if lengths is None else lengths + 1, dropout_p, rng, site)

    mp.setattr(NN, "attention", bad)


MUTANTS = {
    "add-drops-second-grad": (_m_add_drops_b, "bert-padded", {"edges", "stage"}),
    "xent-grad-scale": (_m_xent_scale, "mlp-b200", {"stage"}),
    "ln-grads-swapped": (_m_ln_swap, "bert-s128", {"sequence", "stage"}),
    "packed-pos-plus-one": (_m_pos_plus_one, "bert-packed", {"sequence", "stage"}),
    "pooler-relu": (_m_pool_relu, "bert-s128", {"sequence"}),
    "dropout-bwd-site": (_m_dropout_site, "bert-drop-padded", {"stage"}),
    "bn-eval-in-training": (_m_bn_eval, "resnet-b4", {"sequence"}),
    "mask-lengths-plus-one": (_m_lengths_plus_one, "bert-padded", {"sequence", "stage"}),
}
CASE_BY_ID = {c.id: c for c in CASES}


@gpu
@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_checker_reports_mistake(mutant, monkeypatch):
    mutate, cid, checks = MUTANTS[mutant]
    with pytest.raises(Mismatch) as ei:
        check_case(CASE_BY_ID[cid], monkeypatch, mutate, e2e=False)
    print(f"\n[teeth] {mutant}: {ei.value}")
    assert ei.value.check in checks, str(ei.value)


# ------------------------------------------------------------------------------ LinearXentFn
class _LinearXentBefore(Function):
    """The head as it was before it honoured ``gout``: the reference for gout == 1."""

    @staticmethod
    def forward(ctx, h, w, b, gw, gb, labels, correct):
        h = h.contiguous()
        M, n_cls = h.shape[0], w.shape[0]
        ncp = (n_cls + 7) // 8 * 8
        dl = torch.zeros(M, ncp, device=h.device, dtype=BF16)
        loss = torch.zeros(1, device=h.device, dtype=torch.float32)
        G.gemm_xent(h, w, labels, n_classes=n_cls, bias=b, dlogits=dl, grad_scale=1.0 / M,
                    loss_sum=loss, correct=correct, colsum=gb)
        ctx.save_for_backward(h, w, dl)
        ctx.gw, ctx.n_cls = gw, n_cls
        return loss / M

    @staticmethod
    def backward(ctx, gout):
        h, w, dl = ctx.saved_tensors
        dlv = dl[:, :ctx.n_cls]
        if ctx.gw is not None:
            NN._dw(dlv, h, ctx.gw)
        dh = G.gemm(dlv, w, b_mn=True) if ctx.needs_input_grad[0] else None
        return dh, None, None, None, None, None, None


def _mlp_grads(B, scale=None, fill=None, no_grad=False, seed=4):
    net = nets.MLPNet(784, 256, 62)
    master = make_buffers(net, seed).cuda()
    shadow = master.to(BF16)
    grad = torch.zeros_like(master) if fill is None else fill.clone()
    g = torch.Generator().manual_seed(seed)
    x = net.preprocess(torch.randint(0, 256, (B, 784), generator=g, dtype=torch.uint8).cuda())
    y = torch.randint(0, 62, (B,), generator=g, dtype=torch.int32).cuda()
    b = net.bind(master, shadow, grad)
    if no_grad:
        with torch.no_grad():
            net.loss(b, x, y)
    else:
        loss = net.loss(b, x, y)
        (loss if scale is None else scale * loss).backward()
    torch.cuda.synchronize()
    return grad


@gpu
@pytest.mark.parametrize("c", [2.0, 0.5, -1.0])
def test_linear_xent_scales_with_upstream_gradient(c):
    """(c * loss).backward() gives c times the gradients of loss.backward() for every parameter."""
    g1 = _mlp_grads(200)
    gc = _mlp_grads(200, scale=c)
    net = nets.MLPNet(784, 256, 62)
    V1, Vc = net.spec.views(g1), net.spec.views(gc)
    for name in V1:
        err = float((Vc[name] - c * V1[name]).double().norm())
        assert err <= 2.0 ** -16 * abs(c) * float(V1[name].double().norm()), (name, err)


@gpu
def test_linear_xent_forward_under_no_grad_leaves_grad_untouched():
    net = nets.MLPNet(784, 256, 62)
    fill = torch.randn(net.spec.total, generator=torch.Generator().manual_seed(2)).cuda()
    g = _mlp_grads(200, fill=fill, no_grad=True)
    assert torch.equal(g, fill)


@gpu
def test_linear_xent_gout_one_matches_the_previous_head(monkeypatch):
    """With gout == 1 the gradient buffer is bit for bit what the head computed before it honoured
    gout.  B = 32 rows: every fp32 sum on this path has one atomic per element, so it is deterministic."""
    new = _mlp_grads(32)
    monkeypatch.setattr(NN, "LinearXentFn", _LinearXentBefore)
    old = _mlp_grads(32)
    old2 = _mlp_grads(32)
    assert torch.equal(old, old2), "premise: this shape's gradients are deterministic"
    assert torch.equal(new, old)
