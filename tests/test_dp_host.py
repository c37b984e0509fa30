"""Differentially private aggregation on the host: the config, the Gaussian sampler against the numpy
oracle and fp64 Box-Muller, the C++ ledger against the oracle ledger, snapshots, the device-record DP
word, the heap layout, the accountant, and the DP kernels' register use (ptxas, build.py's flags)."""
import copy
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from bflc_demo_b200 import build
from bflc_demo_b200._native import ledger as _ledger
from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.protocol import oracle as O
from bflc_demo_b200.protocol import privacy

L = _ledger()
RULES = [("fedavg", 1), ("median", 1), ("trimmed_mean", 1)]
BASE = dict(clients=8, committee_size=2, needed_updates=6, aggregate_count=5)
# |z - z_fp64| of the sampler, derived in DESIGN.md ("The Gaussian sampler")
ERROR_BOUND = 3e-6


def same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


# ------------------------------------------------------------------ config
def test_config_accepts_and_rejects():
    c = FLConfig(**BASE).validate()
    assert c.dp_mode == 0 and c.dp_seed is None and c.dp_delta == 1e-5
    assert FLConfig(dp_clip=1.0, **BASE).validate().dp_mode == 1
    assert FLConfig(dp_clip=1.0, dp_noise=0.5, dp_seed=7, **BASE).validate().dp_mode == 2
    assert FLConfig(dp_clip=1.0, aggregation="median", **BASE).validate().dp_mode == 1
    assert FLConfig(dp_clip=1e-45, **BASE).validate().dp_mode == 1           # subnormal, still > 0
    assert FLConfig(dp_clip=1e-46, **BASE).validate().dp_mode == 0           # rounds to 0 in fp32: off
    bad = [dict(dp_clip=-1.0), dict(dp_clip=np.inf), dict(dp_clip=np.nan), dict(dp_clip=1e39),
           dict(dp_clip=1.0, dp_noise=-0.1), dict(dp_clip=1.0, dp_noise=np.inf), dict(dp_clip=1.0, dp_noise=np.nan),
           dict(dp_noise=1.0), dict(dp_clip=1.0, dp_noise=1.0, aggregation="median"),
           dict(dp_clip=1.0, dp_noise=1.0, aggregation="trimmed_mean"), dict(dp_delta=0.0), dict(dp_delta=1.0),
           dict(dp_delta=-1e-5), dict(dp_seed=-1), dict(dp_seed=1 << 64)]
    for kw in bad:
        with pytest.raises(ValueError):
            FLConfig(**{**BASE, **kw}).validate()


def test_config_to_ledger_config_and_env(monkeypatch):
    monkeypatch.setenv("BFLC_DP_CLIP", "0.3")
    monkeypatch.setenv("BFLC_DP_NOISE", "1.1")
    monkeypatch.setenv("BFLC_DP_SEED", "0xFEEDFACECAFEBEEF")
    c = FLConfig.from_env(**BASE)
    assert c.dp_seed == 0xFEEDFACECAFEBEEF and c.dp_mode == 2
    lc = c.to_ledger_config(40)
    assert lc.dp_mode() == 2 and lc.validate() == ""
    assert (lc.dp_clip, lc.dp_noise, lc.dp_seed) == (float(np.float32(0.3)), float(np.float32(1.1)), c.dp_seed)
    assert FLConfig.from_json(c.to_json()) == c
    assert FLConfig(**BASE).to_ledger_config(40).dp_mode() == 0


def test_ledger_config_validation():
    c = L.LedgerConfig()
    assert (c.dp_clip, c.dp_noise, c.dp_seed, c.dp_mode()) == (0.0, 0.0, 0, 0) and c.validate() == ""
    for agg, clip, noise, ok in ((0, 1.0, 0.0, True), (0, 1.0, 2.0, True), (1, 1.0, 0.0, True), (2, 1.0, 0.0, True),
                                 (1, 1.0, 1.0, False), (2, 1.0, 1.0, False), (0, 0.0, 1.0, False),
                                 (0, -1.0, 0.0, False), (0, float("inf"), 0.0, False), (0, float("nan"), 0.0, False),
                                 (0, 1.0, -1.0, False), (0, 1.0, float("nan"), False), (0, 1.0, float("inf"), False)):
        c = L.LedgerConfig()
        c.aggregate_count, c.aggregation, c.trim, c.dp_clip, c.dp_noise = 5, agg, 1, clip, noise
        assert (c.validate() == "") == ok, (agg, clip, noise, c.validate())
        if not ok:
            with pytest.raises(ValueError):
                L.Ledger(c)


def test_run_py_and_sim_reject_bad_dp_flags():
    from bflc_demo_b200 import run
    from bflc_demo_b200.host import sim
    for argv in (["--dp-clip", "-1"], ["--dp-clip", "inf"], ["--dp-noise", "1.0"],
                 ["--dp-clip", "1", "--dp-noise", "-2"], ["--dp-clip", "1", "--dp-noise", "1", "--aggregation", "median"],
                 ["--dp-delta", "0"], ["--dp-delta", "1.5"], ["--dp-seed", "-3"], ["--dp-seed", "notanint"]):
        for main in (run.main, sim.main):
            with pytest.raises(SystemExit) as e:
                main(argv)
            assert e.value.code == 2, (main, argv)


def test_nccl_baseline_refuses_dp():
    from bflc_demo_b200.engine.nccl_baseline import NcclBaselineEngine
    for kw in (dict(dp_clip=1.0), dict(dp_clip=1.0, dp_noise=1.0, dp_seed=1)):
        with pytest.raises(ValueError, match="differentially private"):
            NcclBaselineEngine(FLConfig.for_world(1, **kw), None)


# ------------------------------------------------------------------ the sampler
EDGE = np.array([0, 1, 2, 3, 255, 256, 0xFFFFFF, 0x1000000, 0x1000001, 0x7FFFFFFF, 0x80000000, 0xB504F333,
                 0xFFFFFEFF, 0xFFFFFF00, 0xFFFFFFFD, 0xFFFFFFFE, 0xFFFFFFFF,
                 0x1FFFFFFF, 0x20000000, 0x20000001, 0x3FFFFFFF, 0x40000000, 0x40000001, 0x5FFFFFFF, 0x60000000,
                 0x7FFFFFFE, 0x80000001, 0xBFFFFFFF, 0xC0000000, 0xC0000001, 0xDFFFFFFF, 0xE0000000], np.uint32)


def test_gauss_coordinates_match_the_oracle():
    for seed, epoch, first, n in ((0, 0, 0, 1 << 20), (0x0123456789ABCDEF, 7, 3, 100_003),
                                  ((1 << 64) - 1, (1 << 32) - 1, (1 << 34) + 1, 4097), (42, 1, 0, 1)):
        a, b = L.dp_gauss_coordinates(seed, epoch, first, n), O.dp_gauss(seed, epoch, first, n)
        assert a.dtype == np.float32 and a.shape == (n,) and same(a, b).all(), (seed, epoch, first)
        assert np.isfinite(a).all()
    # a window is the same stream wherever it starts
    full = L.dp_gauss_coordinates(9, 3, 0, 64)
    assert same(L.dp_gauss_coordinates(9, 3, 13, 40), full[13:53]).all()
    assert not same(L.dp_gauss_coordinates(9, 4, 0, 64), full).any()         # the next epoch: other noise
    assert not same(L.dp_gauss_coordinates(10, 3, 0, 64), full).any()        # another seed: other noise


def _edge_words():
    a, b = np.meshgrid(EDGE, EDGE, indexing="ij")
    rng = np.random.default_rng(0)
    low = rng.integers(0, 1 << 32, size=4096, dtype=np.uint64).astype(np.uint32)
    # u1 at its smallest (a = 0) and nearest to 1 (every low byte set), with random angles
    a = np.concatenate([a.ravel(), np.zeros(256, np.uint32), low[:2048] | np.uint32(0xFFFFFF00)])
    b = np.concatenate([b.ravel(), low[2048:2304], low[:2048]])
    return a, b


def test_box_muller_words_match_the_oracle_on_edge_words():
    a, b = _edge_words()
    z0, z1 = L.dp_box_muller_words(a, b)
    o0, o1 = O.dp_box_muller(a, b)
    assert same(z0, o0).all() and same(z1, o1).all()
    assert (np.abs(np.concatenate([z0, z1])) <= np.float32(6.6604369)).all()
    # a = 2^32 - 1: u1 = 1, radius 0; a = 0: u1 = 2^-32, the largest radius sqrt(64 ln 2)
    z0, z1 = L.dp_box_muller_words(np.array([0xFFFFFFFF, 0], np.uint32), np.array([0, 0], np.uint32))
    assert z0[0] == 0 and z1[0] == 0
    assert abs(float(z0[1]) - math.sqrt(64 * math.log(2))) < 4e-6 and z1[1] == 0


def _fp64_box_muller(a, b):
    u = (a.astype(np.float64) + 1.0) / 2.0 ** 32
    r = np.sqrt(-2.0 * np.log(u))
    th = 2.0 * np.pi * b.astype(np.float64) / 2.0 ** 32
    return r * np.cos(th), r * np.sin(th)


def test_box_muller_error_against_fp64():
    rng = np.random.default_rng(11)
    ra = rng.integers(0, 1 << 32, size=1 << 21, dtype=np.uint64).astype(np.uint32)
    rb = rng.integers(0, 1 << 32, size=1 << 21, dtype=np.uint64).astype(np.uint32)
    ea, eb = _edge_words()
    a, b = np.concatenate([ra, ea]), np.concatenate([rb, eb])
    z0, z1 = L.dp_box_muller_words(a, b)
    r0, r1 = _fp64_box_muller(a, b)
    err = max(np.abs(z0 - r0).max(), np.abs(z1 - r1).max())
    assert err <= ERROR_BOUND, err


def test_gauss_is_standard_normal():
    from scipy import stats
    n = 1 << 22
    z = L.dp_gauss_coordinates(0x5EED, 3, 0, n).astype(np.float64)
    assert stats.kstest(z, "norm").pvalue > 1e-3
    # the sample mean has sd 1/sqrt(n) and the sample variance sd sqrt(2/n): 5 sd each
    assert abs(z.mean()) < 5.0 / math.sqrt(n)
    assert abs(z.var() - 1.0) < 5.0 * math.sqrt(2.0 / n)
    # the four normals of one Philox call are uncorrelated
    q = z.reshape(-1, 4)
    c = np.corrcoef(q.T)
    assert np.abs(c - np.eye(4)).max() < 5.0 / math.sqrt(q.shape[0])


# ------------------------------------------------------------------ clipping
def test_clip_coordinates_match_the_oracle():
    rng = np.random.default_rng(3)
    g = rng.standard_normal(1001).astype(np.float32)
    for scale, clip in ((0.01, 1.0), (1.0, 0.5), (10.0, 3.0), (1e-30, 1e-20), (1.0, 1e-40)):
        u = (g + rng.standard_normal(1001).astype(np.float32) * np.float32(scale)).astype(np.float32)
        v, n, s = L.dp_clip_coordinates(g, u, clip)
        ov, on, os_ = O.dp_clip(g, u, clip)
        assert same(v, ov).all() and same([n], [on]).all() and same([s], [os_]).all()
        ref = float(np.sqrt(np.sum((u.astype(np.float64) - g) ** 2)))
        assert abs(n - ref) <= 2 * np.spacing(np.float32(ref))
        if n <= np.float32(clip):
            assert s == 1 and same(v, u).all()                              # unclipped: the upload itself
        else:
            assert s < 1 and np.linalg.norm((v.astype(np.float64) - g)) <= clip * (1 + 1e-5)
    v, n, s = L.dp_clip_coordinates(g, np.full_like(g, np.nan), 1.0)
    assert np.isnan(n) and np.isnan(s) and np.isnan(v).all()


# ------------------------------------------------------------------ ledger vs oracle
def make(agg, trim, *, clip, noise=0.0, seed=0, opt="none", client_num=8, comm=2, aggregate=4, needed=6,
         model_size=37, lr=0.01):
    c = L.LedgerConfig()
    c.client_num, c.comm_count, c.aggregate_count, c.needed_update_count = client_num, comm, aggregate, needed
    c.model_size, c.learning_rate = model_size, lr
    c.aggregation, c.trim = O.AGGREGATIONS.index(agg), trim
    cfg = FLConfig(clients=client_num, committee_size=comm, aggregate_count=aggregate, needed_updates=needed,
                   server_opt=opt, aggregation=agg, trim=trim).validate()
    params = cfg.server_opt_constants
    c.server_opt = cfg.server_opt_id
    c.server_lr, c.server_beta1, c.server_beta2, c.server_tau = (float(params[i]) for i in (0, 1, 2, 5))
    c.dp_clip, c.dp_noise, c.dp_seed = clip, noise, seed
    led = L.Ledger(c)
    orc = O.OracleLedger(client_num, comm, aggregate, needed, lr, model_size, aggregation=agg, trim=trim,
                         server_opt=opt, server_params=params, dp_clip=float(np.float32(clip)),
                         dp_noise=float(np.float32(noise)), dp_seed=seed)
    for i in range(client_num):
        led.RegisterNode(i); orc.RegisterNode(i)
    return led, orc


def one_round(led, orc, rng):
    """Equal sample counts and aggregate_count 4: the FedAvg weights are 1/4, so the ledger's fmaf and the
    oracle's multiply-then-add agree.  Update sizes spread over three decades, so some updates are
    clipped and some are not."""
    ep = led.epoch()
    roles = led.roles()
    trainers = [i for i, r in enumerate(roles) if r & L.ROLE_TRAINER]
    comm = [i for i, r in enumerate(roles) if r & L.ROLE_COMM]
    P = led.config().model_size
    for k, t in enumerate(trainers):
        d = (rng.standard_normal(P) * 10.0 ** (k % 3)).astype(np.float32)
        assert int(led.UploadLocalUpdate(t, d, 100, 0.5, ep)) == orc.UploadLocalUpdate(t, d, 100, 0.5, ep)
    for c in comm:
        row = {t: float(np.float32(rng.random())) for t in trainers}
        led.UploadScores(c, ep, row); orc.UploadScores(c, ep, row)


def check_same(led, orc):
    g, _ = led.QueryGlobalModel()
    assert same(g, orc.global_model).all(), np.flatnonzero(~same(g, orc.global_model))[:8]
    if orc.server_opt != "none":
        m, v = led.server_state()
        assert same(m, orc.server_m).all()
        assert v.size == 0 if orc.server_opt == "momentum" else same(v, orc.server_v).all()


LEDGER_CASES = [(agg, trim, noise, opt) for agg, trim in RULES for noise in (0.0, 1.3) for opt in ("none", "adam")
                if noise == 0.0 or agg == "fedavg"]


@pytest.mark.parametrize("agg,trim,noise,opt", LEDGER_CASES)
def test_ledger_matches_oracle(agg, trim, noise, opt):
    # model changes are lr * delta with |delta| ~ 1, 10, 100 per coordinate over 37 coordinates: norms
    # ~ 0.06, 0.6, 6; a clip of 0.5 clips two of the three kinds
    led, orc = make(agg, trim, clip=0.5, noise=noise, seed=0xABCDEF0123, opt=opt)
    rng = np.random.default_rng(len(agg) * 10 + int(noise) + len(opt))
    for _ in range(4):
        before = orc.global_model.copy()
        one_round(led, orc, rng)
        check_same(led, orc)
        assert not same(before, orc.global_model).all()
        b, h = led.blocks()[-1], orc.history[-1]
        assert b["selected"] == h["selected"] and led.roles() == [orc.role[i] for i in range(8)]
    assert led.verify_chain()


@pytest.mark.parametrize("agg,trim", RULES)
def test_clip_above_every_norm_is_the_ledger_without_dp(agg, trim):
    a, orc_a = make(agg, trim, clip=1e30)
    b, orc_b = make(agg, trim, clip=0.0)
    for r in range(3):
        one_round(a, orc_a, np.random.default_rng(r))
        one_round(b, orc_b, np.random.default_rng(r))
    assert same(a.QueryGlobalModel()[0], b.QueryGlobalModel()[0]).all()
    assert [x["selected"] for x in a.blocks()] == [x["selected"] for x in b.blocks()]
    assert [x["model_hash"] for x in a.blocks()] == [x["model_hash"] for x in b.blocks()]


def test_noise_is_seeded_and_epoch_dependent():
    outs = {}
    for seed in (1, 1, 2):
        led, orc = make("fedavg", 1, clip=0.5, noise=1.0, seed=seed)
        rng = np.random.default_rng(4)
        for _ in range(2):
            one_round(led, orc, rng)
        outs.setdefault(seed, []).append(led.QueryGlobalModel()[0])
    assert same(outs[1][0], outs[1][1]).all() and not same(outs[1][0], outs[2][0]).all()


# ------------------------------------------------------------------ snapshots, hash, device records
def _hdr_end():
    """Byte offset just past the version-4 DP fields: 52-byte v1 header, rule word, optimizer word and
    four floats, DP word and two floats."""
    return 52 + 4 + 4 + 16 + 4 + 8


@pytest.mark.parametrize("noise,opt", [(0.0, "none"), (1.5, "none"), (1.5, "momentum")])
def test_snapshot_v4_round_trip(noise, opt):
    led, orc = make("fedavg", 1, clip=0.5, noise=noise, seed=77, opt=opt)
    one_round(led, orc, np.random.default_rng(5))
    blob = bytes(led.snapshot())
    assert int.from_bytes(blob[4:8], "little") == 4
    assert int.from_bytes(blob[56:60], "little") == O.SERVER_OPTS.index(opt)
    assert int.from_bytes(blob[76:80], "little") == (2 if noise else 1)
    assert np.frombuffer(blob[80:88], np.float32).tolist() == [np.float32(0.5), np.float32(noise)]
    assert (77).to_bytes(8, "little") not in blob[:_hdr_end()]
    back = L.Ledger.restore(blob, dp_seed=77)
    c, c0 = back.config(), led.config()
    assert (c.dp_clip, c.dp_noise, c.dp_seed, c.server_opt) == (c0.dp_clip, c0.dp_noise, 77, c0.server_opt)
    assert back.state_hash() == led.state_hash()
    one_round(back, copy.deepcopy(orc), np.random.default_rng(9))          # the noise stream carries on
    one_round(led, orc, np.random.default_rng(9))
    check_same(back, orc)
    check_same(led, orc)
    assert L.Ledger.restore(blob).config().dp_seed == 0                    # the seed is not in the snapshot


def test_snapshot_dp_off_keeps_versions_1_to_3():
    for agg, opt, version in (("fedavg", "none", 1), ("median", "none", 2), ("fedavg", "adam", 3)):
        led, orc = make(agg, 1, clip=0.0, opt=opt)
        c = L.LedgerConfig()
        c.client_num, c.comm_count, c.aggregate_count, c.needed_update_count = 8, 2, 4, 6
        c.model_size, c.learning_rate, c.aggregation, c.trim = 37, 0.01, O.AGGREGATIONS.index(agg), 1
        cfg = FLConfig(server_opt=opt).validate()
        c.server_opt = cfg.server_opt_id
        p = cfg.server_opt_constants
        c.server_lr, c.server_beta1, c.server_beta2, c.server_tau = (float(p[i]) for i in (0, 1, 2, 5))
        ref = L.Ledger(c)                                # no DP field touched
        for i in range(8):
            ref.RegisterNode(i)
        for x in (led, ref):
            one_round(x, copy.deepcopy(orc), np.random.default_rng(2))
        blob = bytes(led.snapshot())
        assert int.from_bytes(blob[4:8], "little") == version and blob == bytes(ref.snapshot())
        assert led.state_hash() == ref.state_hash()
        assert L.Ledger.restore(blob).config().dp_mode() == 0


def test_restore_rejects_bad_dp_fields():
    led, orc = make("fedavg", 1, clip=0.5, noise=1.0, seed=3)
    one_round(led, orc, np.random.default_rng(4))
    blob = bytes(led.snapshot())
    L.Ledger.restore(blob)
    f32 = lambda x: np.float32(x).tobytes()   # noqa: E731
    bad = []
    for word in (0, 3, 99, 0xFFFFFFFF, 1):                      # mode word (1: clip only, but noise > 0)
        b = bytearray(blob); b[76:80] = word.to_bytes(4, "little"); bad.append(b)
    for off, val in ((80, 0.0), (80, -1.0), (80, np.inf), (80, np.nan), (84, 0.0), (84, -2.0), (84, np.nan)):
        b = bytearray(blob); b[off:off + 4] = f32(val); bad.append(b)
    b = bytearray(blob); b[52:56] = L.agg_word(1, 1).to_bytes(4, "little"); bad.append(b)   # noise under the median
    b = bytearray(blob); b[56:60] = (4).to_bytes(4, "little"); bad.append(b)                 # unknown optimizer
    for b in bad:
        with pytest.raises((RuntimeError, ValueError)):
            L.Ledger.restore(bytes(b))


def test_state_hash_covers_the_dp_fields():
    hashes = set()
    for clip, noise in ((0.0, 0.0), (0.5, 0.0), (0.25, 0.0), (0.5, 1.0), (0.5, 2.0)):
        led, _ = make("fedavg", 1, clip=clip, noise=noise, seed=5)
        hashes.add(led.state_hash())
    assert len(hashes) == 5
    a, _ = make("fedavg", 1, clip=0.5, noise=1.0, seed=5)
    b, _ = make("fedavg", 1, clip=0.5, noise=1.0, seed=6)
    assert a.state_hash() == b.state_hash()                     # the seed stays out (it is the secret)


def test_append_device_round_checks_the_dp_word():
    for agg, trim in RULES[:2]:
        for clip, noise in ((0.0, 0.0), (1.0, 0.0), (1.0, 2.0)):
            if noise and agg != "fedavg":
                continue
            c = L.LedgerConfig()
            c.client_num, c.comm_count, c.aggregate_count, c.needed_update_count = 8, 2, 5, 6
            c.aggregation, c.trim = O.AGGREGATIONS.index(agg), trim
            c.server_opt, c.dp_clip, c.dp_noise = 2, clip, noise
            led = L.Ledger(c)
            roles = [2, 2] + [1] * 6
            led.Bootstrap(roles)
            rec = dict(epoch=0, role_before=roles, role_after=roles, score_rows=[[0.0] * 8] * 8,
                       scored_mask=[0] * 8, n_samples=[1] * 8, avg_cost=[0.0] * 8, admitted_mask=0,
                       selected_mask=0, global_loss=0.0, model_digest=0, weight_by_score=0)
            mode = c.dp_mode()
            word = L.agg_word(c.aggregation, c.trim, 2, mode)
            assert word & 0xFFFFFF == L.agg_word(c.aggregation, c.trim, 2)
            assert (word >> 24) == (0, 1, 3)[mode]                 # bit 24 clip, bit 25 noise
            for other in range(3):
                if other != mode:
                    msg = led.AppendDeviceRound(dict(rec, agg=L.agg_word(c.aggregation, c.trim, 2, other)))
                    assert "differential privacy" in msg, (agg, mode, other, msg)
            assert led.epoch() == 0
            assert led.AppendDeviceRound(dict(rec, agg=word)) == "" and led.epoch() == 1


# ------------------------------------------------------------------ heap layout
def test_heap_layout_unchanged_without_dp():
    from bflc_demo_b200.parallel.layout import HeapLayout
    sz = None
    for P, ring, extra, ss in ((8 * 517, 16, 0, 0), (11_000_000, 256, 8192, 2)):
        a = HeapLayout(P, ring, extra_bytes=extra, server_state=ss)
        b = HeapLayout(P, ring, extra_bytes=extra, server_state=ss, dp=False)
        assert a.offsets == b.offsets and a.total_bytes == b.total_bytes and "dp" not in a.offsets
        c = HeapLayout(P, ring, extra_bytes=extra, server_state=ss, dp=True)
        sz = c.sizes
        assert {n: o for n, o in c.offsets.items() if n != "dp"} == a.offsets
        assert c.offsets["dp"] % 4096 == 0 and c.offsets["dp"] == max(c.offsets.values())
        last = max(o + (P * 4 if n.startswith("server_") else 0) for n, o in a.offsets.items())
        assert c.offsets["dp"] >= last and c.offsets["dp"] + sz["DpPage"] <= c.total_bytes
        assert a.dp_kwargs(0, 1.0, 0.0, 5) == {}
        assert c.dp_kwargs(2, 1.0, 0.5, 5) == dict(dp_mode=2, dp_clip=1.0, dp_noise=0.5, dp_seed=5,
                                                   dp_off=c.offsets["dp"])
    assert sz["FLAG_NORM"] == 32 and sz["FLAG_COUNT"] == 64
    # partials [2][8][8] fp64, norm and scale [8] fp32, sigma, epoch, ticket, pad, block partials [528][8] fp64
    assert sz["DpPage"] == 2 * 8 * 8 * 8 + 2 * 8 * 4 + 4 * 4 + 528 * 8 * 8


# ------------------------------------------------------------------ accountant
def test_epsilon_matches_a_brentq_solution():
    from scipy import optimize, stats
    for z in (0.5, 0.8, 1.0, 1.7, 4.0, 10.0):
        for T in (1, 10, 100, 1000):
            for delta in (1e-3, 1e-5, 1e-8):
                mu = math.sqrt(T) / z

                def f(e):
                    return stats.norm.cdf(-e / mu + mu / 2) - math.exp(e + stats.norm.logcdf(-e / mu - mu / 2)) - delta
                eps = privacy.epsilon(z, T, delta)
                if f(0.0) <= 0:
                    assert eps == 0.0
                    continue
                ref = optimize.brentq(f, 0.0, 2 * eps + 1, xtol=1e-14, rtol=1e-14, maxiter=500)
                assert abs(eps - ref) <= 1e-6 * ref, (z, T, delta, eps, ref)


def test_epsilon_is_below_the_rdp_bound_and_monotone():
    for delta in (1e-3, 1e-5, 1e-9):
        for z in (0.3, 0.7, 1.0, 2.0, 5.0, 20.0):
            prev = -1.0
            for T in (1, 2, 5, 10, 50, 100, 1000, 10_000):
                e = privacy.epsilon(z, T, delta)
                assert e <= privacy.rdp_epsilon(z, T, delta) + 1e-12, (z, T, delta)
                assert e >= prev                                    # more rounds: more epsilon
                prev = e
        for T in (1, 10, 1000):
            es = [privacy.epsilon(z, T, delta) for z in (0.3, 0.7, 1.0, 2.0, 5.0, 20.0)]
            assert all(x >= y for x, y in zip(es, es[1:]))           # more noise: less epsilon
    assert privacy.epsilon(1.0, 0, 1e-5) == 0.0
    assert math.isfinite(privacy.epsilon(0.05, 10_000, 1e-10))     # mu = 2000: no overflow
    with pytest.raises(ValueError):
        privacy.epsilon(0.0, 10, 1e-5)
    with pytest.raises(ValueError):
        privacy.epsilon(1.0, 10, 1.0)


def test_privacy_imports_no_scipy():
    code = "import sys, bflc_demo_b200.protocol.privacy as p; p.epsilon(1.0, 10, 1e-5); assert 'scipy' not in sys.modules"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([os.sys.executable, "-c", code], capture_output=True, text=True, cwd=root,
                       env=dict(os.environ, PYTHONPATH=root))
    assert r.returncode == 0, r.stderr[-2000:]


# ------------------------------------------------------------------ ptxas
def test_dp_kernels_have_no_stack_frame_or_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("no nvcc")
    inc = [f"-I{build.CSRC / d}" for d in ("include", "ledger", "runtime")]
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, *inc, "-c", str(build.CSRC / "kernels" / "fed_kernels.cu"),
           "-o", str(tmp_path / "f.o")]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    log = proc.stdout + proc.stderr
    assert proc.returncode == 0, log[-3000:]
    props = re.findall(r"Function properties for \w*k_consensus_dp(ILb[01]ELi[0-3]ELi[12]EE)\w*\s*\n\s*"
                       r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    found = {inst: (int(a), int(b), int(c)) for inst, a, b, c in props}
    # <kRobust, kServerOpt, kDp>: clip under every rule and optimizer, noise under FedAvg only
    want = {f"ILb{r}ELi{o}ELi{d}EE" for r in (0, 1) for o in range(4) for d in (1, 2) if not (r and d == 2)}
    assert set(found) == want, (sorted(found), log[-3000:])
    assert all(v == (0, 0, 0) for v in found.values()), found
    norms = re.findall(r"Function properties for \w*k_update_norms\w*\s*\n\s*"
                       r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert norms == [("0", "0", "0")], norms
