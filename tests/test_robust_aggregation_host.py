"""Byzantine-robust aggregation on the host: the config, the shared combine function against the
numpy oracle, the C++ ledger against the oracle ledger under each rule, snapshots, the device-record
rule check, and the consensus kernel's register use (ptxas, build.py's flags)."""
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
from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.protocol import oracle as O

L = _ledger()
RULES = [("fedavg", 1), ("median", 1), ("trimmed_mean", 1), ("trimmed_mean", 2)]


def same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


# ------------------------------------------------------------------ config
def test_config_accepts_and_rejects():
    base = dict(clients=8, committee_size=2, needed_updates=6, aggregate_count=6)
    assert FLConfig(**base).validate().aggregation == "fedavg"
    for agg, trim in (("median", 1), ("median", 9), ("trimmed_mean", 1), ("trimmed_mean", 2)):
        c = FLConfig(aggregation=agg, trim=trim, **base).validate()
        assert c.aggregation_rule == O.AGGREGATIONS.index(agg)
    for kw in (dict(aggregation="krum"), dict(aggregation="trimmed_mean", trim=0),
               dict(aggregation="trimmed_mean", trim=3),                 # 2 * 3 == aggregate_count
               dict(aggregation="median", weight_by_score=True),
               dict(aggregation="trimmed_mean", trim=1, weight_by_score=True)):
        with pytest.raises(ValueError):
            FLConfig(**{**base, **kw}).validate()
    FLConfig(weight_by_score=True, **base).validate()                   # FedAvg keeps the score weight


def test_config_from_env_and_ledger_config(monkeypatch):
    monkeypatch.setenv("BFLC_AGGREGATION", "trimmed_mean")
    monkeypatch.setenv("BFLC_TRIM", "2")
    c = FLConfig.from_env(clients=8, committee_size=2, needed_updates=6, aggregate_count=6)
    assert (c.aggregation, c.trim) == ("trimmed_mean", 2)
    lc = c.to_ledger_config(40)
    assert (lc.aggregation, lc.trim) == (2, 2) and lc.validate() == ""
    assert FLConfig.from_json(c.to_json()) == c
    lc = FLConfig(clients=8, committee_size=2, needed_updates=6, aggregate_count=6).to_ledger_config(40)
    assert lc.aggregation == 0


def test_ledger_config_validation():
    c = L.LedgerConfig()                       # 20 / 4 / top-6 of 10
    for agg, trim, ok in ((0, 0, True), (1, 0, True), (2, 1, True), (2, 2, True), (2, 3, False), (2, 0, False),
                          (3, 1, False), (-1, 1, False)):
        c.aggregation, c.trim = agg, trim
        assert (c.validate() == "") == ok, (agg, trim)
    c.aggregation, c.trim, c.weight_by_score = 1, 1, 1
    assert c.validate() != ""
    with pytest.raises(ValueError):
        L.Ledger(c)


# ------------------------------------------------------------------ the combine function
SPECIAL = [np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-40, -1e-40, 1.5, -1.5, 3.4e38, -3.4e38, 1e-45]
NAN_PAYLOADS = [0x7FC00000, 0x7F800001, 0xFFC00000, 0xFFFFFFFF, 0x7FA00123]


@settings(max_examples=300, deadline=None)
@given(n=st.integers(1, 64), p=st.integers(1, 24), trim=st.integers(0, 40), seed=st.integers(0, 2**32 - 1))
def test_aggregate_coordinates_matches_oracle(n, p, trim, seed):
    rng = np.random.default_rng(seed)
    v = (rng.standard_normal((n, p)) * 10.0 ** rng.integers(-3, 4)).astype(np.float32)
    m = rng.random((n, p)) < 0.3
    v[m] = rng.choice(np.array(SPECIAL, np.float32), size=int(m.sum()))
    nanm = rng.random((n, p)) < 0.08
    v.view(np.uint32)[nanm] = rng.choice(np.array(NAN_PAYLOADS, np.uint32), size=int(nanm.sum()))
    if n > 1:                                     # ties
        v[rng.integers(0, n)] = v[rng.integers(0, n)]
    got = L.aggregate_coordinates(v, trim)
    want = O.robust_combine(v, trim)
    assert same(got, want).all(), (v, trim, got, want)


def test_combine_semantics():
    f = np.float32
    assert L.aggregate_coordinates(np.array([[-0.0]], f), 0)[0].tobytes() == f(-0.0).tobytes()   # n = 1: the value
    assert L.aggregate_coordinates(np.array([[-0.0], [0.0]], f), 5)[0] == 0                       # even median
    v = np.array([[1.0], [2.0], [np.nan], [9.0], [-np.inf]], f)
    assert L.aggregate_coordinates(v, 2)[0] == 2.0                   # median: -inf < 1 < 2 < 9 < NaN
    assert L.aggregate_coordinates(v, 1)[0] == f(12.0) / f(3)        # keeps 1, 2, 9
    assert np.isnan(L.aggregate_coordinates(v, 0)[0])
    a, b = f(1.0000001), f(3.3)
    assert L.aggregate_coordinates(np.array([[a], [b]], f), 1)[0] == f(0.5) * (a + b)   # = median_of
    with pytest.raises(ValueError):
        L.aggregate_coordinates(np.zeros((65, 2), f), 1)


# ------------------------------------------------------------------ ledger vs oracle
def make(agg, trim, client_num=8, comm=2, aggregate=5, needed=6, model_size=37):
    c = L.LedgerConfig()
    c.client_num, c.comm_count, c.aggregate_count, c.needed_update_count = client_num, comm, aggregate, needed
    c.model_size, c.learning_rate = model_size, 0.01
    c.aggregation, c.trim = O.AGGREGATIONS.index(agg), trim
    led = L.Ledger(c)
    orc = O.OracleLedger(client_num, comm, aggregate, needed, 0.01, model_size, aggregation=agg, trim=trim)
    for i in range(client_num):
        led.RegisterNode(i); orc.RegisterNode(i)
    return led, orc


def one_round(led, orc, rng, deltas=None):
    ep = led.epoch()
    roles = led.roles()
    trainers = [i for i, r in enumerate(roles) if r & L.ROLE_TRAINER]
    comm = [i for i, r in enumerate(roles) if r & L.ROLE_COMM]
    P = led.config().model_size
    for k, t in enumerate(trainers):
        d = deltas[k] if deltas is not None else rng.standard_normal(P).astype(np.float32)
        if deltas is None and k == 0:
            d[:4] = [np.nan, np.inf, -np.inf, -0.0]
        assert int(led.UploadLocalUpdate(t, d, 100 + t, 0.5, ep)) == orc.UploadLocalUpdate(t, d, 100 + t, 0.5, ep)
    for c in comm:
        row = {t: float(np.float32(rng.random())) for t in trainers}
        led.UploadScores(c, ep, row); orc.UploadScores(c, ep, row)
    return trainers


@pytest.mark.parametrize("agg,trim", RULES)
def test_ledger_matches_oracle(agg, trim):
    led, orc = make(agg, trim)
    rng = np.random.default_rng(11)
    for _ in range(5):
        one_round(led, orc, rng)
        g, _ = led.QueryGlobalModel()
        if agg == "fedavg":     # the ledger sums with fmaf, the oracle with a separate multiply
            np.testing.assert_allclose(g, orc.global_model, rtol=1e-5, atol=1e-7)
        else:                   # robust: one combine procedure, bit for bit
            assert same(g, orc.global_model).all()
        b, h = led.blocks()[-1], orc.history[-1]
        assert b["selected"] == h["selected"] and led.roles() == [orc.role[i] for i in range(8)]
    assert led.verify_chain()


def test_robust_rules_stay_in_the_honest_envelope():
    """aggregate_count = every admitted update, one outlier: median / trimmed mean keep every
    coordinate of the step inside the honest deltas' range, FedAvg leaves it."""
    P = 64
    rng = np.random.default_rng(3)
    honest = rng.standard_normal((5, P)).astype(np.float32)
    outlier = (-50.0 * honest.mean(0) + 40.0).astype(np.float32)
    for agg, trim in RULES[:3]:
        led, orc = make(agg, trim, aggregate=6, needed=6, model_size=P)
        one_round(led, orc, rng, deltas=list(honest) + [outlier])
        assert led.blocks()[-1]["selected"] == [2, 3, 4, 5, 6, 7]
        step = -np.asarray(led.QueryGlobalModel()[0], np.float64) / 0.01     # global was 0: step = combine
        lo, hi = honest.min(0) - 1e-5, honest.max(0) + 1e-5
        inside = bool(((step >= lo) & (step <= hi)).all())
        assert inside == (agg != "fedavg"), agg


# ------------------------------------------------------------------ snapshots and device records
def test_snapshot_versions():
    rng = np.random.default_rng(5)
    led, orc = make("fedavg", 1)
    one_round(led, orc, rng)
    blob = bytes(led.snapshot())
    assert int.from_bytes(blob[4:8], "little") == 1                     # FedAvg: the original format
    back = L.Ledger.restore(blob)
    assert back.config().aggregation == 0 and back.state_hash() == led.state_hash()
    for agg, trim in RULES[1:]:
        led, orc = make(agg, trim)
        one_round(led, orc, rng)
        blob = bytes(led.snapshot())
        assert int.from_bytes(blob[4:8], "little") == 2
        back = L.Ledger.restore(blob)
        c = back.config()
        assert c.aggregation == O.AGGREGATIONS.index(agg)
        assert L.agg_word(c.aggregation, c.trim) == L.agg_word(led.config().aggregation, trim)
        assert back.state_hash() == led.state_hash()
        one_round(back, copy.deepcopy(orc), np.random.default_rng(9))   # keeps aggregating under the rule
        one_round(led, copy.deepcopy(orc), np.random.default_rng(9))
        assert same(back.QueryGlobalModel()[0], led.QueryGlobalModel()[0]).all()
        # the rule word (rule | trim << 8) follows the 52-byte v1 header: a bad rule or trim raises
        for word in (7, 0, 2, 2 | 300 << 8, 1 | 5 << 8, 0xFFFFFFFF):
            bad = bytearray(blob)
            bad[52:56] = word.to_bytes(4, "little")
            with pytest.raises((RuntimeError, ValueError)):
                L.Ledger.restore(bytes(bad))
    # a version-1 blob restores as FedAvg
    led, orc = make("fedavg", 1)
    assert L.Ledger.restore(bytes(led.snapshot())).config().aggregation == 0


def test_append_device_round_checks_the_rule_word():
    for agg, trim in RULES:
        c = L.LedgerConfig()
        c.client_num, c.comm_count, c.aggregate_count, c.needed_update_count = 8, 2, 5, 6
        c.aggregation, c.trim = O.AGGREGATIONS.index(agg), trim
        led = L.Ledger(c)
        roles = [2, 2] + [1] * 6
        led.Bootstrap(roles)
        rec = dict(epoch=0, role_before=roles, role_after=roles, score_rows=[[0.0] * 8] * 8, scored_mask=[0] * 8,
                   n_samples=[1] * 8, avg_cost=[0.0] * 8, admitted_mask=0, selected_mask=0, global_loss=0.0,
                   model_digest=0, weight_by_score=0)
        word = L.agg_word(c.aggregation, c.trim)
        for other in (0, 1, 2 | 1 << 8, 2 | 2 << 8):
            if other != word:
                assert "aggregation rule" in led.AppendDeviceRound(dict(rec, agg=other)), (agg, other)
        if word != 0:
            assert "aggregation rule" in led.AppendDeviceRound(rec)      # no word: a FedAvg record
        assert led.epoch() == 0
        assert led.AppendDeviceRound(dict(rec, agg=word)) == "" and led.epoch() == 1


# ------------------------------------------------------------------ ptxas
def test_consensus_kernel_has_no_stack_frame_or_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("no nvcc")
    inc = [f"-I{build.CSRC / d}" for d in ("include", "ledger", "runtime")]
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, *inc, "-c", str(build.CSRC / "kernels" / "fed_kernels.cu"),
           "-o", str(tmp_path / "f.o")]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    log = proc.stdout + proc.stderr
    assert proc.returncode == 0, log[-3000:]
    props = re.findall(r"Function properties for (\w*k_consensus(ILb[01]E)\w*)\s*\n\s*"
                       r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    found = {inst: (int(a), int(b), int(c)) for _, inst, a, b, c in props}
    assert set(found) == {"ILb0E", "ILb1E"}, log[-3000:]
    assert all(v == (0, 0, 0) for v in found.values()), found
