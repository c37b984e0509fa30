"""Server optimizers (FedAvgM momentum, FedAdam, FedYogi) on the host: the config, the shared step
against the numpy oracle, the C++ ledger against the oracle ledger under each optimizer and rule,
snapshots, the device-record optimizer word, the heap layout, and the consensus kernel's register
use (ptxas, build.py's flags)."""
import copy
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

from bflc_demo_b200 import build
from bflc_demo_b200._native import ledger as _ledger
from bflc_demo_b200.config import SERVER_OPTS, FLConfig
from bflc_demo_b200.protocol import oracle as O

L = _ledger()
OPTS = ["momentum", "adam", "yogi"]
RULES = [("fedavg", 1), ("median", 1), ("trimmed_mean", 1)]


def same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


# ------------------------------------------------------------------ config
def test_config_accepts_and_rejects():
    base = dict(clients=8, committee_size=2, needed_updates=6, aggregate_count=5)
    c = FLConfig(**base).validate()
    assert c.server_opt == "none" and c.server_opt_id == 0 and c.server_state_vectors == 0
    for opt in OPTS:
        c = FLConfig(server_opt=opt, **base).validate()
        assert c.server_opt_id == SERVER_OPTS.index(opt)
        assert c.server_state_vectors == (1 if opt == "momentum" else 2)
        lr, b1, b2, c1, c2, tau = c.server_opt_constants
        assert lr == np.float32(1.0 if opt == "momentum" else 0.01)
        assert (b1, b2, tau) == (np.float32(0.9), np.float32(0.99), np.float32(1e-3))
        assert (c1, c2) == (np.float32(1.0 - float(np.float32(0.9))), np.float32(1.0 - float(np.float32(0.99))))
        assert tuple(np.float32(x) for x in L.server_opt_params(lr, b1, b2, tau)) == c.server_opt_constants
    bad = [dict(server_opt="sgd"), dict(server_opt="adam", server_lr=-1.0), dict(server_opt="adam", server_lr=np.inf),
           dict(server_opt="momentum", server_lr=np.nan), dict(server_opt="momentum", server_beta1=1.0),
           dict(server_opt="yogi", server_beta1=-0.1), dict(server_opt="adam", server_beta2=1.0),
           dict(server_opt="yogi", server_beta2=0.999999999),          # rounds to 1.0 in fp32
           dict(server_opt="adam", server_tau=0.0), dict(server_opt="yogi", server_tau=np.inf),
           dict(server_opt="adam", server_lr=1e39)]                     # overflows fp32
    for kw in bad:
        with pytest.raises(ValueError):
            FLConfig(**{**base, **kw}).validate()
    # momentum ignores beta2 / tau; none ignores every hyperparameter
    FLConfig(server_opt="momentum", server_beta2=5.0, server_tau=0.0, **base).validate()
    FLConfig(server_lr=-1.0, server_beta1=3.0, **base).validate()


def test_config_to_ledger_config_and_env(monkeypatch):
    monkeypatch.setenv("BFLC_SERVER_OPT", "yogi")
    monkeypatch.setenv("BFLC_SERVER_LR", "0.03")
    c = FLConfig.from_env(clients=8, committee_size=2, needed_updates=6, aggregate_count=5)
    lc = c.to_ledger_config(40)
    assert lc.server_opt == 3 and lc.validate() == ""
    assert (lc.server_lr, lc.server_beta1, lc.server_beta2, lc.server_tau) == tuple(
        float(x) for x in np.float32([0.03, 0.9, 0.99, 1e-3]))
    assert FLConfig.from_json(c.to_json()) == c
    assert FLConfig(clients=8, committee_size=2, needed_updates=6, aggregate_count=5).to_ledger_config(40).server_opt == 0


def test_ledger_config_validation():
    c = L.LedgerConfig()
    assert c.server_opt == 0 and c.validate() == ""
    for opt, lr, b1, b2, tau, ok in ((1, 1.0, 0.9, 5.0, 0.0, True), (2, 0.01, 0.9, 0.99, 1e-3, True),
                                     (3, 0.01, 0.0, 0.0, 1e-3, True), (4, 1.0, 0.9, 0.99, 1e-3, False),
                                     (-1, 1.0, 0.9, 0.99, 1e-3, False), (1, 0.0, 0.9, 0.99, 1e-3, False),
                                     (1, float("inf"), 0.9, 0.99, 1e-3, False), (1, 1.0, 1.0, 0.99, 1e-3, False),
                                     (2, 0.01, 0.9, 1.0, 1e-3, False), (3, 0.01, 0.9, -0.5, 1e-3, False),
                                     (2, 0.01, 0.9, 0.99, 0.0, False), (3, 0.01, 0.9, 0.99, float("nan"), False),
                                     (0, -1.0, 7.0, 7.0, -1.0, True)):
        c.server_opt, c.server_lr, c.server_beta1, c.server_beta2, c.server_tau = opt, lr, b1, b2, tau
        assert (c.validate() == "") == ok, (opt, lr, b1, b2, tau)
        if not ok:
            with pytest.raises(ValueError):
                L.Ledger(c)


def test_run_py_rejects_bad_server_flags():
    from bflc_demo_b200 import run
    for argv in (["--server-opt", "nesterov"], ["--server-opt", "adam", "--server-beta2", "1.5"],
                 ["--server-opt", "momentum", "--server-lr", "-2"], ["--server-opt", "yogi", "--server-tau", "0"]):
        with pytest.raises(SystemExit) as e:
            run.main(argv)
        assert e.value.code == 2, argv


def test_nccl_baseline_refuses_a_server_optimizer():
    from bflc_demo_b200.engine.nccl_baseline import NcclBaselineEngine
    with pytest.raises(ValueError, match="server optimizer"):
        NcclBaselineEngine(FLConfig.for_world(1, server_opt="adam"), None)


# ------------------------------------------------------------------ the step
SPECIAL = [np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-40, -1e-40, 1e-45, 1.5, -1.5, 3.4e38, -3.4e38, 1e-20, 1e20]


def _vectors(rng, p):
    out = []
    for _ in range(4):
        x = (rng.standard_normal(p) * 10.0 ** rng.integers(-6, 7)).astype(np.float32)
        m = rng.random(p) < 0.25
        x[m] = rng.choice(np.array(SPECIAL, np.float32), size=int(m.sum()))
        out.append(x)
    return out


@settings(max_examples=300, deadline=None)
@given(opt=st.sampled_from(OPTS), p=st.integers(1, 64), seed=st.integers(0, 2**32 - 1),
       lr=st.sampled_from([1e-30, 1e-6, 0.01, 1.0, 3.0, 1e30]), b1=st.sampled_from([0.0, 0.5, 0.9, 0.999]),
       b2=st.sampled_from([0.0, 0.9, 0.99, 0.9999]), tau=st.sampled_from([1e-38, 1e-8, 1e-3, 1.0]))
def test_server_step_coordinates_matches_oracle(opt, p, seed, lr, b1, b2, tau):
    rng = np.random.default_rng(seed)
    g, a, m, v = _vectors(rng, p)
    if opt != "adam":
        v = np.abs(v)
    if opt == "yogi" and p > 2:              # v == d*d exactly: sign 0 leaves v unchanged
        with np.errstate(all="ignore"):
            d = (g[:2] - a[:2]).astype(np.float32)
            v[:2] = d * d
    params = O.server_constants(lr, b1, b2, tau)
    got = L.server_step_coordinates(g, a, m, v, OPTS.index(opt) + 1, [float(x) for x in params])
    want = O.server_step(g, a, m, v, opt, params)
    for name, x, y in zip(("g", "m", "v"), got, want):
        if name == "v" and opt == "momentum":
            assert same(x, v).all()           # momentum keeps no second moment
            continue
        ok = same(x, y)
        assert ok.all(), (opt, name, np.flatnonzero(~ok)[:4], x[~ok][:4], np.asarray(y)[~ok][:4])


def test_server_step_semantics():
    f = np.float32
    params = O.server_constants(0.5, 0.5, 0.5, 0.25)
    one = lambda opt, g, a, m, v: [x[0] for x in L.server_step_coordinates(   # noqa: E731
        np.array([g], f), np.array([a], f), np.array([m], f), np.array([v], f), OPTS.index(opt) + 1,
        [float(x) for x in params])]
    # momentum: m = 0.5*1 + (3-1) = 2.5, g' = 3 - 0.5*2.5
    assert one("momentum", 3.0, 1.0, 1.0, 0.0)[:2] == [f(1.75), f(2.5)]
    # yogi, v == d*d: sign 0 keeps v; v < d*d grows it, v > d*d shrinks it
    assert one("yogi", 3.0, 1.0, 0.0, 4.0)[2] == f(4.0)
    assert one("yogi", 3.0, 1.0, 0.0, 1.0)[2] == f(1.0 + 0.5 * 4.0)
    assert one("yogi", 3.0, 1.0, 0.0, 8.0)[2] == f(8.0 - 0.5 * 4.0)
    # sign(NaN) is NaN (a (x > 0) - (x < 0) would leave v finite)
    assert np.isnan(one("yogi", 3.0, 1.0, 0.0, np.nan)[2])
    # a subnormal v - d*d is a sign of +-1, not 0 (d*d = 1.8988841e-38, v - d*d ~ 1e-39)
    g_s, a_s = f(2e-19), f(6.219999e-20)
    dd = f(g_s - a_s) * f(g_s - a_s)
    assert 0 < f(2e-38) - dd < np.finfo(f).tiny
    assert one("yogi", g_s, a_s, 0.0, 2e-38)[2] == f(2e-38) - f(0.5) * dd
    # adam: v = 0.5*v + 0.5*d*d, g' = g - (lr*m) / (sqrt(v) + tau)
    g2, m2, v2 = one("adam", 3.0, 1.0, 0.0, 0.0)
    assert (m2, v2) == (f(1.0), f(2.0)) and g2 == f(3.0) - (f(0.5) * f(1.0)) / (np.sqrt(f(2.0)) + f(0.25))
    with pytest.raises(ValueError):
        L.server_step_coordinates(np.zeros(2, f), np.zeros(2, f), np.zeros(2, f), np.zeros(2, f), 0, [1.0] * 6)
    with pytest.raises(ValueError):
        L.server_step_coordinates(np.zeros(2, f), np.zeros(3, f), np.zeros(2, f), np.zeros(2, f), 1, [1.0] * 6)


# ------------------------------------------------------------------ ledger vs oracle
def make(opt, agg, trim, client_num=8, comm=2, aggregate=4, needed=6, model_size=37, lr=0.01, **hp):
    c = L.LedgerConfig()
    c.client_num, c.comm_count, c.aggregate_count, c.needed_update_count = client_num, comm, aggregate, needed
    c.model_size, c.learning_rate = model_size, lr
    c.aggregation, c.trim = O.AGGREGATIONS.index(agg), trim
    cfg = FLConfig(clients=client_num, committee_size=comm, aggregate_count=aggregate, needed_updates=needed,
                   server_opt=opt, **hp).validate()
    params = cfg.server_opt_constants
    c.server_opt = cfg.server_opt_id
    c.server_lr, c.server_beta1, c.server_beta2, c.server_tau = (float(params[i]) for i in (0, 1, 2, 5))
    led = L.Ledger(c)
    orc = O.OracleLedger(client_num, comm, aggregate, needed, lr, model_size, aggregation=agg, trim=trim,
                         server_opt=opt, server_params=params)
    for i in range(client_num):
        led.RegisterNode(i); orc.RegisterNode(i)
    return led, orc


def one_round(led, orc, rng):
    """Equal sample counts and aggregate_count 4: the FedAvg weights are 1/4, so the ledger's fmaf
    and the oracle's multiply-then-add give the same aggregate and the whole step is bit-exact."""
    ep = led.epoch()
    roles = led.roles()
    trainers = [i for i, r in enumerate(roles) if r & L.ROLE_TRAINER]
    comm = [i for i, r in enumerate(roles) if r & L.ROLE_COMM]
    P = led.config().model_size
    for k, t in enumerate(trainers):
        d = (rng.standard_normal(P) * 10.0).astype(np.float32)
        if k == 0:
            d[:3] = [np.inf, -0.0, 1e-40]
        assert int(led.UploadLocalUpdate(t, d, 100, 0.5, ep)) == orc.UploadLocalUpdate(t, d, 100, 0.5, ep)
    for c in comm:
        row = {t: float(np.float32(rng.random())) for t in trainers}
        led.UploadScores(c, ep, row); orc.UploadScores(c, ep, row)


def check_same(led, orc):
    g, _ = led.QueryGlobalModel()
    m, v = led.server_state()
    assert same(g, orc.global_model).all(), np.flatnonzero(~same(g, orc.global_model))[:8]
    assert same(m, orc.server_m).all()
    if orc.server_opt == "momentum":
        assert v.size == 0
    else:
        assert same(v, orc.server_v).all()


@pytest.mark.parametrize("agg,trim", RULES)
@pytest.mark.parametrize("opt", OPTS)
def test_ledger_matches_oracle(opt, agg, trim):
    led, orc = make(opt, agg, trim)
    assert [x.size for x in led.server_state()] == [0, 0]      # allocated on the first host aggregation
    rng = np.random.default_rng(OPTS.index(opt) * 10 + len(agg))
    for _ in range(4):
        one_round(led, orc, rng)
        check_same(led, orc)
        b, h = led.blocks()[-1], orc.history[-1]
        assert b["selected"] == h["selected"] and led.roles() == [orc.role[i] for i in range(8)]
    assert led.verify_chain()


def test_fedavg_nan_poisons_state_but_a_robust_rule_does_not():
    """Under FedAvg one selected NaN makes m NaN for good; the median drops it."""
    out = {}
    for agg in ("fedavg", "median"):
        led, orc = make("momentum", agg, 1, aggregate=4)
        rng = np.random.default_rng(1)
        ep = led.epoch()
        trainers = [i for i, r in enumerate(led.roles()) if r & L.ROLE_TRAINER]
        for k, t in enumerate(trainers):
            d = rng.standard_normal(37).astype(np.float32)
            if k == 0:
                d[5] = np.nan
            led.UploadLocalUpdate(t, d, 100, 0.5, ep)
        for c in (0, 1):
            led.UploadScores(c, ep, {t: 1.0 for t in trainers})     # ties: the lowest ranks, trainer 2 included
        assert trainers[0] in led.blocks()[-1]["selected"]
        out[agg] = bool(np.isnan(led.server_state()[0][5]))
    assert out == {"fedavg": True, "median": False}


def test_none_is_the_existing_update():
    """server_opt none keeps global -= lr * aggregate (not momentum with b1 = 0, lr = 1)."""
    a, orc = make("none", "fedavg", 1)
    c = L.LedgerConfig()
    c.client_num, c.comm_count, c.aggregate_count, c.needed_update_count = 8, 2, 4, 6
    c.model_size, c.learning_rate = 37, 0.01
    b = L.Ledger(c)
    for i in range(8):
        b.RegisterNode(i)
    for led in (a, b):
        one_round(led, copy.deepcopy(orc), np.random.default_rng(3))
    assert same(a.QueryGlobalModel()[0], b.QueryGlobalModel()[0]).all()
    assert a.state_hash() == b.state_hash() and bytes(a.snapshot()) == bytes(b.snapshot())
    assert [x.size for x in a.server_state()] == [0, 0]


# ------------------------------------------------------------------ snapshots, hash, device records
def _hdr_end(blob):
    """Byte offset just past the version-3 hyperparameters (52-byte v1 header + rule word + optimizer
    word + four floats)."""
    return 52 + 4 + 4 + 16


@pytest.mark.parametrize("opt", OPTS)
def test_snapshot_v3_round_trip(opt):
    led, orc = make(opt, "median", 1)
    blob0 = bytes(led.snapshot())                       # before any host aggregation: empty state
    assert int.from_bytes(blob0[4:8], "little") == 3
    back0 = L.Ledger.restore(blob0)
    assert [x.size for x in back0.server_state()] == [0, 0] and back0.state_hash() == led.state_hash()
    rng = np.random.default_rng(5)
    one_round(led, orc, rng)
    blob = bytes(led.snapshot())
    assert int.from_bytes(blob[4:8], "little") == 3
    assert int.from_bytes(blob[52:56], "little") == L.agg_word(1, 1)          # the rule word, always
    assert int.from_bytes(blob[56:60], "little") == OPTS.index(opt) + 1
    back = L.Ledger.restore(blob)
    c, c0 = back.config(), led.config()
    assert (c.server_opt, c.server_lr, c.server_beta1, c.server_beta2, c.server_tau) == (
        c0.server_opt, c0.server_lr, c0.server_beta1, c0.server_beta2, c0.server_tau)
    assert back.state_hash() == led.state_hash()
    for x, y in zip(back.server_state(), led.server_state()):
        assert same(x, y).all() and x.size == y.size
    one_round(back, copy.deepcopy(orc), np.random.default_rng(9))         # the state carries on
    one_round(led, orc, np.random.default_rng(9))
    check_same(back, orc)
    check_same(led, orc)
    # a FedAvg ledger with an optimizer is version 3 too, its rule word 0
    led, _ = make(opt, "fedavg", 1)
    blob = bytes(led.snapshot())
    assert int.from_bytes(blob[4:8], "little") == 3 and int.from_bytes(blob[52:56], "little") == 0
    assert L.Ledger.restore(blob).config().server_opt == OPTS.index(opt) + 1


def test_snapshot_none_keeps_versions_1_and_2():
    for agg, version in (("fedavg", 1), ("median", 2)):
        led, orc = make("none", agg, 1)
        c = L.LedgerConfig()
        c.client_num, c.comm_count, c.aggregate_count, c.needed_update_count = 8, 2, 4, 6
        c.model_size, c.learning_rate, c.aggregation, c.trim = 37, 0.01, O.AGGREGATIONS.index(agg), 1
        ref = L.Ledger(c)                                # a default-config ledger: no optimizer fields touched
        for i in range(8):
            ref.RegisterNode(i)
        for x in (led, ref):
            one_round(x, copy.deepcopy(orc), np.random.default_rng(2))
        blob = bytes(led.snapshot())
        assert int.from_bytes(blob[4:8], "little") == version and blob == bytes(ref.snapshot())
        assert L.Ledger.restore(blob).config().server_opt == 0


def test_restore_rejects_bad_optimizer_fields():
    led, orc = make("adam", "fedavg", 1)
    one_round(led, orc, np.random.default_rng(4))
    blob = bytes(led.snapshot())
    L.Ledger.restore(blob)
    f32 = lambda x: np.float32(x).tobytes()   # noqa: E731
    bad = []
    for word in (0, 4, 99, 0xFFFFFFFF):                                      # optimizer word
        b = bytearray(blob); b[56:60] = word.to_bytes(4, "little"); bad.append(b)
    for off, val in ((60, 0.0), (60, np.inf), (64, 1.0), (68, 1.0), (72, 0.0), (72, np.nan)):   # lr b1 b2 tau
        b = bytearray(blob); b[off:off + 4] = f32(val); bad.append(b)
    # state vector lengths: epoch (4 bytes), global (8-byte length + 37 floats), then m's length word
    m_len = _hdr_end(blob) + 4 + 8 + 37 * 4
    assert int.from_bytes(blob[m_len:m_len + 8], "little") == 37
    for n in (36, 38):
        b = bytearray(blob); b[m_len:m_len + 8] = n.to_bytes(8, "little"); bad.append(b)
    # m present, v dropped (the v vector replaced by an empty one: the blob shrinks by 37 floats)
    v_len = m_len + 8 + 37 * 4
    b = bytearray(blob); b[v_len:v_len + 8 + 37 * 4] = (0).to_bytes(8, "little"); bad.append(b)
    for b in bad:
        with pytest.raises((RuntimeError, ValueError)):
            L.Ledger.restore(bytes(b))


def test_state_hash_covers_the_server_state():
    led, orc = make("momentum", "fedavg", 1)
    one_round(led, orc, np.random.default_rng(6))
    h = led.state_hash()
    blob = bytearray(led.snapshot())
    m_off = _hdr_end(blob) + 4 + 8 + 37 * 4 + 8                           # first float of m
    blob[m_off:m_off + 4] = (np.frombuffer(bytes(blob[m_off:m_off + 4]), np.float32) + np.float32(1)).tobytes()
    other = L.Ledger.restore(bytes(blob))
    assert same(other.QueryGlobalModel()[0], led.QueryGlobalModel()[0]).all()
    assert other.state_hash() != h


def test_append_device_round_checks_the_optimizer_word():
    for opt in ["none"] + OPTS:
        for agg, trim in RULES[:2]:
            c = L.LedgerConfig()
            c.client_num, c.comm_count, c.aggregate_count, c.needed_update_count = 8, 2, 5, 6
            c.aggregation, c.trim = O.AGGREGATIONS.index(agg), trim
            c.server_opt = SERVER_OPTS.index(opt)
            led = L.Ledger(c)
            roles = [2, 2] + [1] * 6
            led.Bootstrap(roles)
            rec = dict(epoch=0, role_before=roles, role_after=roles, score_rows=[[0.0] * 8] * 8,
                       scored_mask=[0] * 8, n_samples=[1] * 8, avg_cost=[0.0] * 8, admitted_mask=0,
                       selected_mask=0, global_loss=0.0, model_digest=0, weight_by_score=0)
            word = L.agg_word(c.aggregation, c.trim, c.server_opt)
            assert word & 0xFFFF == L.agg_word(c.aggregation, c.trim) and word >> 16 == c.server_opt
            for o in range(4):
                other = L.agg_word(c.aggregation, c.trim, o)
                if other != word:
                    assert "server optimizer" in led.AppendDeviceRound(dict(rec, agg=other)), (opt, agg, o)
            assert led.epoch() == 0
            assert led.AppendDeviceRound(dict(rec, agg=word)) == "" and led.epoch() == 1


# ------------------------------------------------------------------ heap layout
def test_heap_layout_unchanged_without_server_state():
    from bflc_demo_b200.parallel.layout import HeapLayout
    for P, ring, extra in ((8 * 517, 16, 0), (11_000_000, 256, 8192)):
        a, b = HeapLayout(P, ring, extra_bytes=extra), HeapLayout(P, ring, extra_bytes=extra, server_state=0)
        assert a.offsets == b.offsets and a.total_bytes == b.total_bytes and "server_m" not in a.offsets
        for k in (1, 2):
            c = HeapLayout(P, ring, extra_bytes=extra, server_state=k)
            assert {n: o for n, o in c.offsets.items() if n in a.offsets} == a.offsets
            names = ("server_m", "server_v")[:k]
            assert set(c.offsets) - set(a.offsets) == set(names)
            ends = sorted((o, o + (P * 4 if n in names else 0)) for n, o in c.offsets.items())
            assert all(o % 4096 == 0 for n, o in c.offsets.items() if n in names)
            assert c.offsets[names[0]] >= a.offsets["extra"] + extra and ends[-1][1] <= c.total_bytes
        assert HeapLayout(P, ring, server_state=1).server_opt_kwargs(0, (1.0,) * 6) == {}


# ------------------------------------------------------------------ ptxas
def test_consensus_instantiations_have_no_stack_frame_or_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("no nvcc")
    inc = [f"-I{build.CSRC / d}" for d in ("include", "ledger", "runtime")]
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, *inc, "-c", str(build.CSRC / "kernels" / "fed_kernels.cu"),
           "-o", str(tmp_path / "f.o")]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    log = proc.stdout + proc.stderr
    assert proc.returncode == 0, log[-3000:]
    props = re.findall(r"Function properties for \w*k_consensus(ILb[01]ELi[0-3]EE)\w*\s*\n\s*"
                       r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    found = {inst: (int(a), int(b), int(c)) for inst, a, b, c in props}
    want = {f"ILb{r}ELi{o}EE" for r in (0, 1) for o in range(4)}      # <kRobust, kServerOpt>
    assert set(found) == want, (sorted(found), log[-3000:])
    assert all(v == (0, 0, 0) for v in found.values()), found
