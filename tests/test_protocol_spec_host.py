"""CPU: exact host models of the round protocol kernels (``csrc/kernels/fed_kernels.cu``,
``fed_admit.cuh``, ``epi::mx8_unpack_unit``) that ``test_gpu_protocol_conformance.py`` checks every
rank's device state against, and the fixtures it runs them on.

* ``plan_model``: what ``k_plan`` writes into a rank's ``RoundPlan`` (candidate list, per-layer
  ``GemmDynamic`` with absolute bias / flag pointers, blob pointers, cleared accumulators, step words).
* ``admission``: first-K-wins tickets -- rank 0's ticket word and every replica's slot words for a
  given upload order.
* ``digest`` / ``two_shot_slices``: the model digest sum of bits(v_i) * ((2i + 1) * 0x9E3779B97F4A7C15)
  mod 2^64, and the even float4 slices two-shot consensus reduces.
* ``byz_upload``: the byzantine upload as this build compiles it -- ``FADD.FTZ d = w - g`` then
  ``FFMA.FTZ out = -d * s + g`` (one rounding, subnormals flushed) -- and ``avg_cost_bound``: the
  ``MUFU.RCP`` + ``FMUL.FTZ`` the division ``loss_sum / n`` becomes under ``--use_fast_math``.
* ``unpack_model``: what ``k_pull_blob`` writes for a candidate blob, through ``ops/mx8.py``.
* ``exact_mlp`` / ``fp64_counts``: integer MLPs with a unique argmax per row, so the validation
  counts are exact for any summation order.

The tests below show that each of eight plausible kernel mistakes changes a checked output of these
fixtures, so the GPU suite would catch it."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from bflc_demo_b200.ops.mx8 import MX8, quantize_mx8_reference
from test_mx8_spec_host import scale_rows
from test_optim_spec_host import f32_fma, f32_sub, same_bits

TRAINER, COMM = 1, 2
KMAX = 8
FLAG_TRAINED, FLAG_SCORED, FLAG_DONE, FLAG_SLICE = 0, 8, 16, 24
GOLDEN = 0x9E3779B97F4A7C15
M64 = (1 << 64) - 1


# ------------------------------------------------------------------ plan and admission
def first_k(roles, n_needed) -> bool:
    """admit::first_k: some trainers will not be awaited."""
    n_tr = sum(1 for r in roles if r & TRAINER)
    return n_needed != 0 and n_needed < n_tr


def plan_model(*, rank, roles, epoch, n_needed, layers, staged, bases, lay, steps, prev,
               stage_master=0, blobs=None, mutant=None) -> dict:
    """RoundPlan of ``rank`` after k_plan.  ``lay``: heap offsets (HeapLayout.offsets + n_params);
    ``prev``: the plan words k_plan reads back (cand_rank, round_seq, opt_total); ``blobs``: None or
    (stage_blob, blob_bytes, upq_off).  Pointers are absolute integers (0 = null)."""
    par = epoch & 1
    trainers = [r for r, x in enumerate(roles) if x & TRAINER]
    cand = list(prev["cand_rank"])
    n_cand = len(trainers)
    cand[:n_cand] = trainers
    fk = first_k(roles, n_needed)
    if fk:
        n_cand, cand = n_needed, [-1] * KMAX
    me = bases[rank]
    out = dict(is_trainer=int(bool(roles[rank] & TRAINER)), is_comm=int(bool(roles[rank] & COMM)), parity=par,
               n_cand=n_cand, cand_rank=cand, dyn=[])
    for off, use in layers:
        d = dict(active=n_cand if out["is_comm"] else 0, wait_value=epoch + 1, map_index=[], bias=[], wait_flag=[])
        li = len(out["dyn"])
        for z in range(KMAX):
            t = cand[z] if z < n_cand and cand[z] >= 0 else 0
            d["map_index"].append(li * KMAX + z if staged else (li * 2 + par) * KMAX + t)
            if staged and stage_master and mutant != "bias_rank0":
                src = stage_master + 4 * z * lay["n_params"]
            else:
                src = bases[t] + lay[f"upload_master{par}"]
            d["bias"].append(src + 4 * off if use else 0)
            d["wait_flag"].append(0 if staged else me + lay["flags"] + 4 * (FLAG_TRAINED + t))
        out["dyn"].append(d)
    cb = []
    for z in range(KMAX):
        t = cand[z] if z < n_cand and cand[z] >= 0 else rank
        if blobs is None:
            cb.append(0)
        else:
            stage, nbytes, upq = blobs
            cb.append(stage + z * nbytes if staged else bases[t] + upq[par])
    out["cand_blob"] = cb
    out.update(correct=[0] * KMAX, loss_sum=0.0, train_correct=0, upload_blocks=0, consensus_blocks=0,
               digest_acc=0, step_barrier=0, round_seq=(prev["round_seq"] + 1) & 0xFFFFFFFF,
               opt_step=prev["opt_total"], opt_total=prev["opt_total"] + (steps if out["is_trainer"] else 0))
    return out


def admission(order, K, epoch):
    """Trainers upload in ``order`` (each takes one ticket): rank 0's ticket word, the slot words every
    replica holds, and the admitted ranks (the first K, in ticket order)."""
    tag = (epoch + 1) << 8
    return tag | len(order), {z: tag | order[z] for z in range(K)}, list(order[:K])


def slot_trainers(roles, n_needed, order, mutant=None):
    """Trainer rank of each candidate slot: ticket order in first-K mode, ascending rank otherwise."""
    trainers = [r for r, x in enumerate(roles) if x & TRAINER]
    if first_k(roles, n_needed) and mutant != "ascending":
        return list(order[:n_needed])
    return trainers[: n_needed] if first_k(roles, n_needed) else trainers


def pull_model(shadows, slots, par, mutant=None):
    """k_pull: staging slot z = the bf16 upload shadow of parity par of slot z's trainer
    (shadows[(rank, parity)] = uint16 array)."""
    p = 1 - par if mutant == "parity" else par
    return [shadows[(t, p)] for t in slots]


# ------------------------------------------------------------------ digest
def digest(v, base: int = 0, mutant=None) -> int:
    """sum_i bits(v_i) * ((2 (base + i) + 1) * GOLDEN) mod 2^64 over fp32 v."""
    bits = np.ascontiguousarray(v, np.float32).view(np.uint32).astype(np.uint64)
    idx = np.arange(base, base + bits.size, dtype=np.uint64)
    mul = idx if mutant == "digest_idx" else idx * np.uint64(2) + np.uint64(1)
    with np.errstate(over="ignore"):
        return int(np.sum(bits * (mul * np.uint64(GOLDEN)), dtype=np.uint64))


def two_shot_slices(P: int, R: int, mutant=None):
    """Element ranges [lo, hi) each rank reduces in two-shot mode: float4 slices rounded up to even."""
    nv = P // 4
    per = (nv + R - 1) // R
    if mutant != "odd_slices":
        per += per & 1
    out = []
    for r in range(R):
        lo = min(per * r, nv)
        out.append((4 * lo, 4 * min(lo + per, nv)))
    return out


def slice_digests(model, R, mutant=None):
    return [digest(model[lo:hi], lo) for lo, hi in two_shot_slices(model.size, R, mutant)]


# ------------------------------------------------------------------ upload arithmetic
def byz_upload(w, g, s, mutant=None):
    """k_upload's byzantine value: d = w - g (FADD.FTZ), out = fma(-d, s, g) (FFMA.FTZ)."""
    d = f32_sub(w, g)
    if mutant == "unfused":
        with np.errstate(over="ignore", invalid="ignore"):
            return f32_sub(g, (d * np.float32(s)).astype(np.float32))
    return f32_fma(-d, np.float32(s), g)


def avg_cost_bound(loss, n):
    """(centre, bound) of loss / max(n, 1) as MUFU.RCP (at most 1 ulp off 1/n) then FMUL.FTZ (0.5 ulp):
    |got - loss/n| <= 2^-22 |loss/n| + 2^-126, and exact when n is a power of two."""
    q = float(np.float32(loss)) / max(n, 1)
    if (max(n, 1) & (max(n, 1) - 1)) == 0 and (q == 0 or abs(q) >= 2.0 ** -126):
        return q, 0.0
    return q, 2.0 ** -22 * abs(q) + 2.0 ** -126


# ------------------------------------------------------------------ MXFP8 blob unpack
def mlp_blob_layout(in_dim, hidden):
    """Mx8MlpLayout (the GPU suite asserts it equals mx8_mlp_layout)."""
    kb1, kb2, rb1 = (in_dim + 127) // 128, (hidden + 127) // 128, (hidden + 127) // 128
    cur, out = 0, {}
    for name, nbytes in (("w1q", hidden * in_dim), ("w1sf", rb1 * kb1 * 512), ("w2q", 64 * hidden),
                         ("w2sf", kb2 * 512), ("b1", hidden * 4), ("b2", 256)):
        out[name] = cur
        cur += (nbytes + 127) // 128 * 128
    out.update(total=cur, kb1=kb1, kb2=kb2)
    return out


def blob_model(w1, b1, w2, b2, in_dim, hidden, nc):
    """What quantize_mlp_blob writes (the regions the unpack reads): uint8 [total]."""
    L = mlp_blob_layout(in_dim, hidden)
    blob = np.zeros(L["total"], np.uint8)
    r1 = quantize_mx8_reference(torch.as_tensor(w1, dtype=torch.float32).reshape(hidden, in_dim))
    w2p = torch.zeros(64, hidden)
    w2p[:nc] = torch.as_tensor(w2, dtype=torch.float32).reshape(nc, hidden)
    r2 = quantize_mx8_reference(w2p)
    blob[L["w1q"]:L["w1q"] + hidden * in_dim] = r1.q.view(torch.uint8)[:, :in_dim].reshape(-1).numpy()
    n1 = r1.sf.numel()
    blob[L["w1sf"]:L["w1sf"] + min(n1, L["w2q"] - L["w1sf"])] = r1.sf.numpy()[: L["w2q"] - L["w1sf"]]
    blob[L["w2q"]:L["w2q"] + 64 * hidden] = r2.q.view(torch.uint8)[:, :hidden].reshape(-1).numpy()
    blob[L["w2sf"]:L["w2sf"] + L["kb2"] * 512] = r2.sf.numpy()[: L["kb2"] * 512]
    blob[L["b1"]:L["b1"] + 4 * hidden] = np.asarray(b1, np.float32).view(np.uint8)
    bb2 = np.zeros(64, np.float32)
    bb2[:nc] = b2
    blob[L["b2"]:L["b2"] + 256] = bb2.view(np.uint8)
    return blob


def _dequant(blob, qo, so, rows, K, nkb, n_rb, mutant):
    q = torch.from_numpy(blob[qo:qo + rows * K].copy()).view(torch.float8_e4m3fn).reshape(rows, K)
    sf = torch.from_numpy(blob[so:so + n_rb * nkb * 512].copy())
    if mutant != "neighbour_scale":
        return MX8(q, sf, rows, K).dequantize()
    s = scale_rows(sf, n_rb * 128, K)[:rows].long()               # [rows, groups]
    col = torch.arange(K)
    grp = col // 32 + ((col % 32) >= 16).long()                    # second 16-half: the next group's byte
    e = s[:, grp.clamp(max=s.shape[1] - 1)]
    return q.float() * torch.exp2(e.double() - 127).float()


def unpack_model(blob, in_dim, hidden, nc, w1_off, w2_off, stage_dq, stage_blob, mutant=None):
    """k_pull_blob for one slot: the dequantised W1 [hidden, in_dim] and the first nc rows of W2 as bf16
    into stage_dq (uint16, flat parameter layout), b1 | b2 (hidden + 64 floats) copied into stage_blob
    at the blob's b1 offset.  Returns new arrays; everything else keeps its bytes."""
    L = mlp_blob_layout(in_dim, hidden)
    dq, sb = stage_dq.copy(), stage_blob.copy()
    w1 = _dequant(blob, L["w1q"], L["w1sf"], hidden, in_dim, L["kb1"], (hidden + 127) // 128, mutant)
    rows2 = 64 if mutant == "w2_all_rows" else nc
    w2 = _dequant(blob, L["w2q"], L["w2sf"], 64, hidden, L["kb2"], 1, mutant)[:rows2]
    for w, off in ((w1, w1_off), (w2, w2_off)):
        h = w.to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16).reshape(-1)
        n = min(h.size, dq.size - off)                             # (a mistake may run past the slot)
        dq[off:off + n] = h[:n]
    n = 4 * (hidden + 64)
    sb[L["b1"]:L["b1"] + n] = blob[L["b1"]:L["b1"] + n]
    return dq, sb


# ------------------------------------------------------------------ exact validation fixtures
def exact_mlp(seed, in_dim, hidden, nc, spec):
    """Flat fp32 master of an MLP whose validation is exact: W1 / W2 in {-1, 0, 1}, integer b1,
    b2 = integer + a distinct multiple of 1/128 per class (no two logits of a row tie)."""
    rng = np.random.default_rng(seed)
    m = np.zeros(spec.total, np.float32)
    o = {e.name: e.offset for e in spec.entries}
    m[o["w1"]:o["w1"] + hidden * in_dim] = rng.integers(-1, 2, hidden * in_dim)
    m[o["b1"]:o["b1"] + hidden] = rng.integers(-4, 5, hidden)
    m[o["w2"]:o["w2"] + nc * hidden] = rng.integers(-1, 2, nc * hidden)
    m[o["b2"]:o["b2"] + nc] = rng.integers(-4, 5, nc) + rng.permutation(128)[:nc] / 128.0
    return m


def val_inputs(seed, n_val, in_dim):
    rng = np.random.default_rng(seed)
    return (rng.random((n_val, in_dim)) < 0.25).astype(np.float32)


def fp64_predictions(x, weights_master, bias_master, spec, hidden, nc):
    """argmax of relu(x W1^T + b1) W2^T + b2 in fp64, weights of one model, biases of another."""
    o = {e.name: e.offset for e in spec.entries}
    in_dim = x.shape[1]
    w1 = weights_master[o["w1"]:o["w1"] + hidden * in_dim].astype(np.float64).reshape(hidden, in_dim)
    w2 = weights_master[o["w2"]:o["w2"] + nc * hidden].astype(np.float64).reshape(nc, hidden)
    b1 = bias_master[o["b1"]:o["b1"] + hidden].astype(np.float64)
    b2 = bias_master[o["b2"]:o["b2"] + nc].astype(np.float64)
    h = np.maximum(x.astype(np.float64) @ w1.T + b1, 0.0)
    assert h.max() < 256                                          # exact in bf16
    lg = h @ w2.T + b2
    if nc > 1:
        top2 = np.sort(lg, axis=1)[:, -2:]
        assert (top2[:, 1] > top2[:, 0]).all()
    return lg.argmax(1)


def labels_for(seed, preds, nc):
    """Labels: each row is some model's prediction or random, so every model scores in between."""
    rng = np.random.default_rng(seed)
    pick = rng.integers(0, len(preds) + 1, preds[0].size)
    lab = rng.integers(0, nc, preds[0].size)
    for i, p in enumerate(preds):
        lab = np.where(pick == i, p, lab)
    return lab.astype(np.int32)


# Shared fixtures of the GPU suite
E2E = dict(in_dim=784, hidden=256, nc=62, n_val=256, R=6, n_comm=2)
BYZ_SCALES = (5.0, 1.7)


def byz_fixture(P, seed):
    """(w, g): random values plus fp32 subnormals, +-0, +-inf and NaN payloads."""
    rng = np.random.default_rng(seed)
    g = (rng.standard_normal(P) * 0.5).astype(np.float32)
    w = (g + rng.standard_normal(P).astype(np.float32) * 0.1).astype(np.float32)
    spec = np.array([0x00000001, 0x80000005, 0x007FFFFF, 0x00000000, 0x80000000, 0x7F800000, 0xFF800000,
                     0x7FC00001, 0xFFA12345, 0x7F7FFFFF, 0x00800000, 0x3F800001], np.uint32).view(np.float32)
    w[:spec.size] = spec
    g[spec.size:2 * spec.size] = spec
    w[2 * spec.size:3 * spec.size] = spec
    g[2 * spec.size:3 * spec.size] = spec[::-1]
    return w, g


# ------------------------------------------------------------------ tests
def test_digest_matches_python_integers():
    rng = np.random.default_rng(1)
    v = rng.standard_normal(1003).astype(np.float32)
    want = sum(int(b) * (((2 * (7 + i) + 1) * GOLDEN) & M64) for i, b in enumerate(v.view(np.uint32))) & M64
    assert digest(v, 7) == want
    P, R = 8 * 517, 3
    assert sum(slice_digests(v[:P] if v.size >= P else np.resize(v, P), R)) & M64 == digest(np.resize(v, P))


def test_two_shot_slices_cover_the_model_with_even_float4_slices():
    for P, R in ((8 * 517, 2), (8 * 517, 3), (8 * 517, 8), (8, 8), (4096, 5)):
        s = two_shot_slices(P, R)
        assert s[0][0] == 0 and s[-1][1] == P
        for (a, b), (c, _) in zip(s, s[1:]):
            assert b == c and (a // 4) % 2 == 0


def test_byz_model_is_one_rounding_and_flushes():
    w = np.array([3.0, 1e-39, 2.0], np.float32)
    g = np.array([1.0, 0.0, 1e-39], np.float32)
    out = byz_upload(w, g, 5.0)
    assert out[0] == np.float32(1.0 - 5.0 * 2.0)
    assert out[1] == 0.0 and not np.signbit(out[1])              # subnormal w flushed before the subtraction
    assert out[2] == np.float32(-10.0)                             # d = 2 - 0 (g flushed), out = -5 d + 0


def test_avg_cost_bound_is_exact_for_powers_of_two():
    assert avg_cost_bound(3.5, 8) == (3.5 / 8, 0.0)
    c, b = avg_cost_bound(1.0, 3)
    assert b > 0 and abs(c - 1 / 3) < 1e-15


def test_admission_words():
    ticket, slots, adm = admission([5, 2, 7, 3], 2, 4)
    assert ticket == (5 << 8) | 4 and slots == {0: (5 << 8) | 5, 1: (5 << 8) | 2} and adm == [5, 2]


def test_blob_model_round_trips_through_the_decoder():
    from bflc_demo_b200.models.mlp import mlp_spec
    for in_dim, hidden, nc in ((64, 256, 10), (112, 128, 1), (1008, 288, 64)):
        spec = mlp_spec(in_dim, hidden, nc)
        o = {e.name: e.offset for e in spec.entries}
        m = torch.randn(spec.total, generator=torch.Generator().manual_seed(in_dim)).numpy()
        w1 = m[:hidden * in_dim].reshape(hidden, in_dim)
        w2 = m[o["w2"]:o["w2"] + nc * hidden].reshape(nc, hidden)
        blob = blob_model(w1, m[o["b1"]:o["b1"] + hidden], w2, m[o["b2"]:o["b2"] + nc], in_dim, hidden, nc)
        dq, _ = unpack_model(blob, in_dim, hidden, nc, o["w1"], o["w2"], np.zeros(spec.total, np.uint16),
                             np.zeros(blob.size, np.uint8))
        want = quantize_mx8_reference(torch.from_numpy(w1.copy())).dequantize().to(torch.bfloat16)
        got = torch.from_numpy(dq[:hidden * in_dim].view(np.int16).copy()).view(torch.bfloat16).reshape(hidden, in_dim)
        assert torch.equal(got, want)


# -------------------------------------------------------------- teeth: every mistake fails a fixture
def _e2e_models():
    from bflc_demo_b200.models.mlp import mlp_spec
    p = E2E
    spec = mlp_spec(p["in_dim"], p["hidden"], p["nc"])
    models = {r: exact_mlp(100 + r, p["in_dim"], p["hidden"], p["nc"], spec) for r in range(p["R"])}
    return spec, models


def _mutant_fails(mutant) -> bool:
    p = E2E
    if mutant in ("parity", "ascending"):
        roles = [COMM, COMM, TRAINER, TRAINER, TRAINER, TRAINER]
        order = [4, 2, 5, 3]
        shadows = {(t, q): np.full(4, 16 * t + q, np.uint16) for t in range(6) for q in (0, 1)}
        ok = slot_trainers(roles, 2, order)
        bad = slot_trainers(roles, 2, order, mutant)
        right = pull_model(shadows, ok, 1)
        wrong = pull_model(shadows, bad, 1, mutant)
        return any(not np.array_equal(a, b) for a, b in zip(right, wrong))
    if mutant == "bias_rank0":
        spec, models = _e2e_models()
        x = val_inputs(7, p["n_val"], p["in_dim"])
        for t in (4, 2):                                           # the first-K fixture's admitted trainers
            own = fp64_predictions(x, models[t], models[t], spec, p["hidden"], p["nc"])
            stale = fp64_predictions(x, models[t], models[0], spec, p["hidden"], p["nc"])
            if (own != stale).any():
                return True
        return False
    if mutant == "digest_idx":
        v = np.random.default_rng(3).standard_normal(8 * 517).astype(np.float32)
        return digest(v) != digest(v, mutant=mutant)
    if mutant == "odd_slices":
        v = np.random.default_rng(3).standard_normal(8 * 517).astype(np.float32)
        return slice_digests(v, 3) != slice_digests(v, 3, mutant) or slice_digests(v, 8) != slice_digests(v, 8, mutant)
    if mutant in ("neighbour_scale", "w2_all_rows"):
        from bflc_demo_b200.models.mlp import mlp_spec
        for in_dim, hidden, nc in ((64, 256, 10), (112, 128, 1)):
            spec = mlp_spec(in_dim, hidden, nc)
            o = {e.name: e.offset for e in spec.entries}
            g = torch.Generator().manual_seed(5)
            w1 = (torch.randn(hidden, in_dim, generator=g) * torch.logspace(-3, 3, in_dim)).numpy()
            w2 = (torch.randn(nc, hidden, generator=g) * torch.logspace(-3, 3, hidden)).numpy()
            blob = blob_model(w1, np.ones(hidden), w2, np.ones(nc), in_dim, hidden, nc)
            canary = np.full(spec.total, 0xABCD, np.uint16)
            sb = np.full(blob.size, 0xCD, np.uint8)
            a = unpack_model(blob, in_dim, hidden, nc, o["w1"], o["w2"], canary, sb)
            b = unpack_model(blob, in_dim, hidden, nc, o["w1"], o["w2"], canary, sb, mutant)
            if not all(np.array_equal(u, v) for u, v in zip(a, b)):
                return True
        return False
    if mutant == "unfused":
        w, g = byz_fixture(4096, 11)
        return any(not same_bits(byz_upload(w, g, s), byz_upload(w, g, s, mutant)).all() for s in BYZ_SCALES)
    raise AssertionError(mutant)


MUTANTS = ["parity", "ascending", "bias_rank0", "digest_idx", "odd_slices", "neighbour_scale", "w2_all_rows",
           "unfused"]


@pytest.mark.parametrize("mutant", MUTANTS)
def test_teeth_every_modelled_mistake_fails_a_fixture(mutant):
    assert _mutant_fails(mutant), f"the fixtures cannot tell the {mutant!r} mistake from the kernel"
