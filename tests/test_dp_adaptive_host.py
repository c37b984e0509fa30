"""Adaptive clipping of DP-FedAvg on the CPU: dp_exp, the clip update and the noise split against numpy and
fp64, convergence to the target quantile, the C++ ledger against the oracle, snapshots, the hash, the
device-record check, config / CLI refusals, the heap layout, the site word, ptxas, and modelled mistakes."""
from __future__ import annotations

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
F = np.float32
SEED = 0xC11D5EED


def same(a, b):
    a, b = np.asarray(a, F), np.asarray(b, F)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


# ------------------------------------------------------------------ dp_exp, the update, the split
def _exp_args():
    dense = np.linspace(-O.DP_EXP_MAX, O.DP_EXP_MAX, 1 << 20, dtype=F)
    ln2 = math.log(2.0)
    # the clamp bounds, +-0, and the reduction boundaries (k + 1/2) ln 2 with their neighbours
    edges = [O.DP_EXP_MAX, -O.DP_EXP_MAX, 0.0, -0.0, 1e-30, -1e-30, 2.0 ** -126, -2.0 ** -149]
    for k in range(-6, 6):
        b = F((k + 0.5) * ln2)
        if abs(b) <= O.DP_EXP_MAX:
            edges += [b, np.nextafter(b, F(np.inf)), np.nextafter(b, F(-np.inf))]
    return np.concatenate([dense, np.array(edges, F)])


# |dp_exp(x) / e^x - 1|: Horner's 8 roundings and the final scale (9 u), the reduced argument's two
# roundings times |x| <= 4 plus the polynomial's truncation (< 6e-9) -- under 2e-6
EXP_BOUND = 2e-6


def test_dp_exp_host_matches_numpy_and_fp64():
    x = _exp_args()
    host, ref = L.dp_exp_values(x), O.dp_exp(x)
    assert same(host, ref).all(), x[~same(host, ref)][:8]
    rel = np.abs(host.astype(np.float64) / np.exp(x.astype(np.float64)) - 1.0)
    assert rel.max() <= EXP_BOUND, (rel.max(), x[np.argmax(rel)])
    assert host[np.where(x == 0)[0]].tolist() == [1.0, 1.0]                 # +0 and -0
    assert (host > 0).all() and np.isfinite(host).all()


def test_clip_update_matches_fp64_geometric_update():
    rng = np.random.default_rng(1)
    for _ in range(4000):
        n = int(rng.integers(1, 9))
        b = int(rng.integers(0, n + 1))
        count = F(b + rng.standard_normal() * 2.0)
        clip = F(10.0 ** rng.uniform(-6, 6))
        q, lr = F(rng.uniform(0.05, 0.95)), F(rng.uniform(0.01, 2.0))
        got = L.dp_clip_next(clip, count, n, q, lr)
        assert same(got, O.dp_clip_next(clip, count, n, q, lr))
        x = -float(lr) * (float(count) / n - float(q))
        x = min(max(x, -O.DP_EXP_MAX), O.DP_EXP_MAX)
        want = float(clip) * math.exp(x)
        # the exponent's three roundings (|x| <= 4: 3 u 4), dp_exp, and the final product
        assert abs(got / want - 1.0) <= 12 * 2.0 ** -24 + EXP_BOUND + 2.0 ** -24, (got, want)
    # the clip stays a finite, positive normal float whatever the count
    assert L.dp_clip_next(O.DP_CLIP_MIN, 1e30, 1, 0.5, 100.0) == O.DP_CLIP_MIN
    assert L.dp_clip_next(O.DP_CLIP_MAX, -1e30, 1, 0.5, 100.0) == O.DP_CLIP_MAX
    assert L.dp_clip_next(1.0, 0.0, 4, 0.5, 0.2) > 1.0 > L.dp_clip_next(1.0, 4.0, 4, 0.5, 0.2)


def test_noise_split_matches_and_keeps_the_total_multiplier():
    for z, sb in ((1.0, 2.0), (0.7, 5.0), (3.0, 1.6), (1.1, 0.5501)):
        zd = privacy.noise_split(z, sb)
        assert zd == L.dp_noise_split(z, sb)
        # z_delta^-2 + (2 sigma_b)^-2 = z^-2, up to the fp32 rounding of z_delta
        tot = 1.0 / math.sqrt(zd ** -2 + (2.0 * float(F(sb))) ** -2)
        assert abs(tot / float(F(z)) - 1.0) <= 2.0 ** -23
    with pytest.raises(ValueError):
        privacy.noise_split(3.0, 1.4)                                          # not > z / 2
    # epsilon is a function of the total multiplier only
    assert privacy.epsilon(1.0, 50, 1e-5) == privacy.epsilon(float(F(1.0)), 50, 1e-5)


def test_noised_count_matches_the_host_sampler_and_is_keyed_by_epoch():
    for epoch in range(64):
        for b, n in ((0, 3), (2, 3), (5, 5)):
            got = L.dp_noised_count(b, n, 1.5, SEED, epoch)
            xi = O.dp_gauss(SEED, epoch, 0, 1, O.DP_CLIP_SITE)[0]
            assert same(got, O.dp_noised_count(b, n, 1.5, SEED, epoch))
            assert same(got, F(F(b) + F(F(1.5) * xi)))
    assert L.dp_noised_count(2, 3, 0.0, SEED, 4) == 2.0                      # clip only: b exactly
    assert L.dp_noised_count(0, 0, 1.5, SEED, 4) == 0.0                      # empty round: nothing drawn
    xs = [O.dp_gauss(SEED, e, 0, 1, O.DP_CLIP_SITE)[0] for e in range(200)]
    assert len(set(np.asarray(xs, F).tolist())) == 200 and abs(np.mean(xs)) < 0.3


def test_site_word_is_distinct():
    sites = {O.DP_SITE, O.DPSGD_SITE, O.DPSGD_SAMPLE_SITE}
    assert O.DP_CLIP_SITE == L.DP_CLIP_SITE and O.DP_CLIP_SITE not in sites and O.DP_CLIP_SITE >= 1 << 24
    # its stream is not the aggregate's coordinate 0..3 of the same (seed, epoch)
    assert not same(O.dp_gauss(SEED, 3, 0, 1, O.DP_CLIP_SITE), O.dp_gauss(SEED, 3, 0, 4)[:1]).any()


@pytest.mark.parametrize("start", [0.01, 100.0])
def test_clip_converges_to_the_quantile(start):
    """sigma_b = 0, 8 norms a round from a fixed log-normal law: from 100x below and 100x above the median,
    C_t is within 15 % of the true 0.5-quantile after 120 rounds and stays there (averaged over the last 40)."""
    rng = np.random.default_rng(7)
    q, lr, med = 0.5, 0.2, 1.0                                     # median of exp(N(0, 0.5^2)) is 1
    clip = F(start * med)
    traj = []
    for t in range(160):
        norms = np.exp(rng.standard_normal(8) * 0.5).astype(F)
        _, clip = O.dp_clip_round(norms, clip, q, lr, 0.0, 0, t)
        traj.append(float(clip))
    assert abs(traj[119] / med - 1) < 0.5 and abs(np.mean(traj[120:]) / med - 1) < 0.15, traj[110:]
    # the clip moves by at most e^(lr * max(q, 1 - q)) per round
    steps = np.abs(np.diff(np.log(traj)))
    assert steps.max() <= lr * max(q, 1 - q) + 1e-5


# ------------------------------------------------------------------ ledger vs oracle
def make(agg, *, clip, noise=0.0, quantile=0.5, lr=0.2, count_noise=0.0, seed=SEED, opt="none", trim=1,
         learning_rate=0.01):
    c = L.LedgerConfig()
    c.client_num, c.comm_count, c.aggregate_count, c.needed_update_count = 8, 2, 4, 6
    c.model_size, c.learning_rate = 37, learning_rate
    c.aggregation, c.trim = O.AGGREGATIONS.index(agg), trim
    cfg = FLConfig(clients=8, committee_size=2, aggregate_count=4, needed_updates=6, server_opt=opt,
                   aggregation=agg, trim=trim).validate()
    params = cfg.server_opt_constants
    c.server_opt = cfg.server_opt_id
    c.server_lr, c.server_beta1, c.server_beta2, c.server_tau = (float(params[i]) for i in (0, 1, 2, 5))
    c.dp_clip, c.dp_noise, c.dp_seed = clip, noise, seed
    c.dp_clip_quantile, c.dp_clip_lr, c.dp_count_noise = quantile, lr, count_noise
    led = L.Ledger(c)
    orc = O.OracleLedger(8, 2, 4, 6, learning_rate, 37, aggregation=agg, trim=trim, server_opt=opt, server_params=params,
                         dp_clip=float(F(clip)), dp_noise=float(F(noise)), dp_seed=seed,
                         dp_clip_quantile=float(F(quantile)), dp_clip_lr=float(F(lr)),
                         dp_count_noise=float(F(count_noise)))
    for i in range(8):
        led.RegisterNode(i); orc.RegisterNode(i)
    return led, orc


def one_round(led, orc, rng):
    """Equal sample counts, 4 selected: FedAvg weights 1/4.  Model changes lr * delta with norms ~ 0.06, 0.6, 6."""
    ep = led.epoch()
    roles = led.roles()
    trainers = [i for i, r in enumerate(roles) if r & L.ROLE_TRAINER]
    comm = [i for i, r in enumerate(roles) if r & L.ROLE_COMM]
    for k, t in enumerate(trainers):
        d = (rng.standard_normal(37) * 10.0 ** (k % 3)).astype(F)
        assert int(led.UploadLocalUpdate(t, d, 100, 0.5, ep)) == orc.UploadLocalUpdate(t, d, 100, 0.5, ep)
    for c in comm:
        row = {t: float(F(rng.random())) for t in trainers}
        led.UploadScores(c, ep, row); orc.UploadScores(c, ep, row)


CASES = [(agg, noise, opt) for agg in ("fedavg", "median", "trimmed_mean") for noise in (0.0, 1.3)
         for opt in ("none", "momentum", "adam", "yogi") if noise == 0.0 or agg == "fedavg"]


@pytest.mark.parametrize("agg,noise,opt", CASES)
def test_ledger_matches_oracle(agg, noise, opt):
    led, orc = make(agg, clip=0.5, noise=noise, count_noise=1.0 if noise else 0.0, opt=opt)
    rng = np.random.default_rng(len(agg) + int(noise * 10) + len(opt))
    clips = []
    for _ in range(12):
        one_round(led, orc, rng)
        g, _ = led.QueryGlobalModel()
        assert same(g, orc.global_model).all()
        clip, count, n_sel = led.last_clip_step()
        h = orc.history[-1]
        assert same(clip, h["clip"]) and same(count, h["count"]) and n_sel == h["n_sel"] == 4
        assert same(led.dp_clip_now(), orc.clip_now)
        clips.append(clip)
        if noise == 0:
            assert count == int(count) and 0 <= count <= 4
    assert len(set(clips)) >= 4                                    # the clip really moves
    assert led.verify_chain()


# ------------------------------------------------------------------ a norm equal to the clip, modelled mistakes
def exact_round(led, orcs):
    """One round whose four selected updates have lr * delta norms 0.5, 0.005, 0.005 and 50 (lr 0.5: the first is
    exactly 0.5 = C_0, delta = e_0); the committee scores pick exactly these four of the six trainers."""
    ep = led.epoch()
    roles = led.roles()
    trainers = [i for i, r in enumerate(roles) if r & L.ROLE_TRAINER]
    comm = [i for i, r in enumerate(roles) if r & L.ROLE_COMM]
    scale = [(0, 1.0), (1, 0.01), (2, 0.01), (3, 100.0), (4, 1000.0), (5, 1000.0)]
    for t, (j, a) in zip(trainers, scale):
        d = np.zeros(37, F)
        d[j] = a
        for x in (led, *orcs):
            assert int(x.UploadLocalUpdate(t, d, 100, 0.5, ep)) == 0
    row = {t: float(F(0.9 - 0.1 * k)) for k, t in enumerate(trainers)}
    for c in comm:
        for x in (led, *orcs):
            x.UploadScores(c, ep, row)
    return [trainers[k] for k in range(4)]


def test_ledger_counts_a_norm_equal_to_the_clip():
    for noise, sb in ((0.0, 0.0), (1.3, 1.0)):
        led, orc = make("fedavg", clip=0.5, noise=noise, count_noise=sb, learning_rate=0.5)
        sel = exact_round(led, [orc])
        assert led.blocks()[-1]["selected"] == sorted(sel)
        clip, count, n_sel = led.last_clip_step()
        # b = 3: the update at exactly C is not clipped, so it is counted
        assert (clip, n_sel) == (0.5, 4) and same(count, L.dp_noised_count(3, 4, sb, SEED, 0))
        if noise == 0:
            assert count == 3.0
        h = orc.history[-1]
        assert same(count, h["count"]) and same(led.dp_clip_now(), orc.clip_now)
        assert same(led.QueryGlobalModel()[0], orc.global_model).all()


def _count(norms, clip, strict=False):
    key = lambda v: int(np.array(F(v)).view(np.uint32))   # noqa: E731
    return sum(1 for v in norms if (key(v) < key(clip) if strict else key(v) <= key(clip)))


def _mistaken_round(mistake, K):
    """``oracle.dp_clip_round`` with one modelled mistake (K: the configured aggregate_count)."""
    def step(norms, clip, quantile, lr, count_noise, seed, epoch):
        c, n = F(clip), len(norms)
        if n == 0:
            return F(0), (O.dp_clip_next(c, F(0), 1, quantile, lr) if mistake == "empty_updates" else c)
        cnt = O.dp_noised_count(_count(norms, c, strict=mistake == "strict"), n, count_noise, seed,
                                0 if mistake == "epoch_free" else epoch)
        nxt = O.dp_clip_next(c, cnt, K if mistake == "divide_by_K" else n, quantile, lr)
        if mistake == "count_after_update":
            cnt = O.dp_noised_count(_count(norms, nxt), n, count_noise, seed, epoch)
            nxt = O.dp_clip_next(c, cnt, n, quantile, lr)
        return cnt, nxt
    return step


def _host_fixture(model, noise, sb, monkeypatch):
    """Host rounds through Ledger::aggregate_locked (the exact-norm round, then three random ones) against the
    oracle with ``model`` in place of its clip step: True when every round agrees bit for bit."""
    led, orc = make("fedavg", clip=0.5, noise=noise, count_noise=sb, learning_rate=0.5)
    rng = np.random.default_rng(3)
    agree = True
    with monkeypatch.context() as mp:
        model(mp)
        for r in range(4):
            if r == 0:
                exact_round(led, [orc])
            else:
                one_round(led, orc, rng)
            clip, count, n_sel = led.last_clip_step()
            h = orc.history[-1]
            agree &= bool(same(count, h["count"]) and same(led.dp_clip_now(), orc.clip_now)
                          and same(led.QueryGlobalModel()[0], orc.global_model).all())
    return agree


def _device_fixtures(step):
    """Device records through Ledger::AppendDeviceRound: a round that selects 2 of aggregate_count 3 (norms 0.5 and
    2.0 at C = 1), and a round that selects nothing.  True when ``step`` gives the ledger's C_{t+1} for both."""
    agree = True
    for admitted, norms in ((0b0110, [F(0.5), F(2.0)]), (0, [])):
        led, rec = _device_ledger(1.3, 1.0)
        n = len(norms)
        count = L.dp_noised_count(_count(norms, F(1.0)), n, 1.0, SEED, 0)
        rec = dict(rec, admitted_mask=admitted, selected_mask=admitted, scored_mask=[admitted, 0, 0, 0],
                   role_after=[1, 2, 1, 1] if admitted else [2, 1, 1, 1], clip=1.0, count=float(count), n_sel=n)
        assert led.AppendDeviceRound(rec) == "", rec
        want = led.dp_clip_now()
        if n == 0:
            assert want == 1.0 and count == 0.0                  # an empty round keeps C and draws nothing
        agree &= bool(same(step(norms, F(1.0), 0.5, 0.2, 1.0, SEED, 0)[1], want))
    return agree


MISTAKES = {
    "z_not_split": lambda mp: mp.setattr(privacy, "noise_split", lambda z, sb: float(F(z))),
    "count_after_update": None, "strict": None, "divide_by_K": None, "epoch_free": None, "empty_updates": None,
}


@pytest.mark.parametrize("mistake", list(MISTAKES))
def test_modelled_mistakes_are_caught(mistake, monkeypatch):
    """Every fixture runs through the C++ ledger: host rounds (clip only and with noise) and device records.  The
    oracle agrees with the ledger on all of them, and the oracle with the modelled mistake disagrees on one."""
    correct = lambda mp: None   # noqa: E731
    patch = MISTAKES[mistake] or (lambda mp: mp.setattr(O, "dp_clip_round", _mistaken_round(mistake, 4)))
    for noise, sb in ((0.0, 0.0), (1.3, 1.0)):
        assert _host_fixture(correct, noise, sb, monkeypatch)
    assert _device_fixtures(O.dp_clip_round)
    caught = not all(_host_fixture(patch, noise, sb, monkeypatch) for noise, sb in ((0.0, 0.0), (1.3, 1.0)))
    if mistake != "z_not_split":
        caught |= not _device_fixtures(_mistaken_round(mistake, 3))
    assert caught, mistake


# ------------------------------------------------------------------ snapshots, hash, device records
def test_snapshot_v5_round_trip_and_v4_unchanged():
    led, orc = make("fedavg", clip=0.5, noise=1.3, count_noise=1.0, seed=77)
    for r in range(3):
        one_round(led, orc, np.random.default_rng(r))
    blob = bytes(led.snapshot())
    assert int.from_bytes(blob[4:8], "little") == 5
    hdr = 52 + 4 + 4 + 16 + 4 + 8                      # the version-4 header
    q, lr, sb, cnow = np.frombuffer(blob[hdr:hdr + 16], F)
    assert (q, lr, sb) == (F(0.5), F(0.2), F(1.0)) and same(cnow, led.dp_clip_now())
    back = L.Ledger.restore(blob, dp_seed=77)
    assert back.state_hash() == led.state_hash() and same(back.dp_clip_now(), led.dp_clip_now())
    one_round(back, copy.deepcopy(orc), np.random.default_rng(9))       # the trajectory carries on
    one_round(led, orc, np.random.default_rng(9))
    assert same(back.QueryGlobalModel()[0], orc.global_model).all() and same(back.dp_clip_now(), orc.clip_now)
    # adaptive off: the version-4 blob is the one a ledger that never heard of the new fields writes
    a, oa = make("fedavg", clip=0.5, noise=1.3, quantile=0.0, seed=77)
    c = L.LedgerConfig()
    c.client_num, c.comm_count, c.aggregate_count, c.needed_update_count = 8, 2, 4, 6
    c.model_size, c.learning_rate = 37, 0.01
    c.server_opt, c.server_lr = 0, a.config().server_lr
    c.dp_clip, c.dp_noise, c.dp_seed = 0.5, 1.3, 77
    ref = L.Ledger(c)
    for i in range(8):
        ref.RegisterNode(i)
    for x in (a, ref):
        one_round(x, copy.deepcopy(oa), np.random.default_rng(2))
    assert int.from_bytes(bytes(a.snapshot())[4:8], "little") == 4
    assert bytes(a.snapshot()) == bytes(ref.snapshot()) and a.state_hash() == ref.state_hash()


def test_restore_rejects_bad_adaptive_fields():
    led, orc = make("fedavg", clip=0.5)
    one_round(led, orc, np.random.default_rng(4))
    blob = bytes(led.snapshot())
    hdr = 52 + 4 + 4 + 16 + 4 + 8
    L.Ledger.restore(blob)
    bad = []
    for off, val in ((0, 0.0), (0, 1.0), (0, -0.5), (0, np.nan), (4, 0.0), (4, np.inf), (8, 1.0),
                     (12, 0.0), (12, -1.0), (12, np.inf), (12, np.nan)):
        b = bytearray(blob); b[hdr + off:hdr + off + 4] = F(val).tobytes(); bad.append(b)
    for b in bad:
        with pytest.raises((RuntimeError, ValueError)):
            L.Ledger.restore(bytes(b))


def test_state_hash_covers_the_adaptive_fields():
    hashes = set()
    for q, lr, sb in ((0.0, 0.2, 0.0), (0.5, 0.2, 1.0), (0.4, 0.2, 1.0), (0.5, 0.3, 1.0), (0.5, 0.2, 2.0)):
        led, _ = make("fedavg", clip=0.5, noise=1.3, quantile=q, lr=lr, count_noise=sb)
        hashes.add(led.state_hash())
    assert len(hashes) == 5
    a, oa = make("fedavg", clip=0.5)
    b, ob = make("fedavg", clip=0.5)
    one_round(a, oa, np.random.default_rng(3)); one_round(b, ob, np.random.default_rng(3))
    assert a.state_hash() == b.state_hash()
    one_round(a, oa, np.random.default_rng(4)); one_round(b, ob, np.random.default_rng(5))
    assert a.dp_clip_now() != b.dp_clip_now() and a.state_hash() != b.state_hash()


def _device_ledger(noise=0.0, sb=0.0):
    c = L.LedgerConfig()
    c.client_num, c.comm_count, c.aggregate_count, c.needed_update_count = 4, 1, 3, 3
    c.dp_clip, c.dp_noise, c.dp_seed = 1.0, noise, SEED
    c.dp_clip_quantile, c.dp_clip_lr, c.dp_count_noise = 0.5, 0.2, sb
    led = L.Ledger(c)
    roles = [2, 1, 1, 1]
    led.Bootstrap(roles)
    rows = [[0.0, 0.9, 0.8, 0.7]] + [[0.0] * 4] * 3
    rec = dict(epoch=0, role_before=roles, role_after=[1, 2, 1, 1],
               score_rows=rows, scored_mask=[0b1110, 0, 0, 0], n_samples=[1] * 4, avg_cost=[0.0] * 4,
               admitted_mask=0b1110, selected_mask=0b1110, global_loss=0.0, model_digest=0, weight_by_score=0,
               agg=L.agg_word(0, 1, 0, c.dp_kernel_mode()))
    return led, rec


def test_append_device_round_flags_a_tampered_clip_record():
    for noise, sb in ((0.0, 0.0), (1.3, 1.0)):
        led, rec = _device_ledger(noise, sb)
        good = L.dp_noised_count(2, 3, sb, SEED, 0)
        for clip, count, n_sel in ((F(0.5), good, 3), (F(1.0), good, 2), (F(1.0), F(good) + F(0.25), 3),
                                   (F(1.0), F(7.0) if sb == 0 else F(good) + F(1e-3), 3)):
            msg = led.AppendDeviceRound(dict(rec, clip=float(clip), count=float(count), n_sel=n_sel))
            assert "clip trajectory mismatch" in msg, (clip, count, n_sel, msg)
        assert "clip trajectory mismatch" in led.AppendDeviceRound(rec)                 # no clip record
        assert led.epoch() == 0 and led.dp_clip_now() == 1.0
        assert led.AppendDeviceRound(dict(rec, clip=1.0, count=float(good), n_sel=3)) == ""
        assert same(led.dp_clip_now(), L.dp_clip_next(1.0, good, 3, 0.5, 0.2))
        # the word carries the adaptive bit: a fixed-clip record is refused
        led2, rec2 = _device_ledger(noise, sb)
        fixed = L.agg_word(0, 1, 0, 2 if noise else 1)
        assert "differential privacy" in led2.AppendDeviceRound(dict(rec2, agg=fixed, clip=1.0, count=float(good), n_sel=3))
    assert L.agg_word(0, 1, 0, 3) >> 24 == 0b101 and L.agg_word(0, 1, 0, 4) >> 24 == 0b111


# ------------------------------------------------------------------ config, CLI, baseline, layout
def test_config_accepts_and_refuses():
    ok = [dict(dp_clip=1.0, dp_clip_quantile=0.5), dict(dp_clip=1.0, dp_clip_quantile=0.9, dp_clip_lr=1.0),
          dict(dp_clip=1.0, dp_noise=1.0, dp_clip_quantile=0.5, dp_count_noise=0.6),
          dict(dp_clip=1.0, dp_clip_quantile=0.5, aggregation="median"),
          dict(dp_clip=1.0, dp_clip_quantile=0.5, aggregation="trimmed_mean", trim=1, aggregate_count=4),
          dict(dp_clip=1.0, dp_clip_quantile=0.5, server_opt="adam")]
    for kw in ok:
        c = FLConfig(**kw).validate()
        assert c.dp_adaptive and c.to_ledger_config(10).dp_adaptive()
    bad = [dict(dp_clip_quantile=0.5), dict(dp_clip=1.0, dp_clip_quantile=1.0), dict(dp_clip=1.0, dp_clip_quantile=-0.1),
           dict(dp_clip=1.0, dp_clip_quantile=0.5, dp_clip_lr=0.0), dict(dp_clip=1.0, dp_clip_quantile=0.5, dp_clip_lr=np.inf),
           dict(dp_clip=1.0, dp_clip_quantile=0.5, dp_count_noise=1.0),
           dict(dp_clip=1.0, dp_noise=1.0, dp_clip_quantile=0.5, dp_count_noise=0.5),
           dict(dp_clip=1.0, dp_noise=1.0, dp_clip_quantile=0.5),
           dict(dp_clip=1.0, dp_count_noise=1.0), dict(dp_clip=1.0, dp_clip_quantile=np.nan)]
    for kw in bad:
        with pytest.raises(ValueError):
            FLConfig(**kw).validate()
        c = L.LedgerConfig()
        c.dp_clip, c.dp_noise = float(kw.get("dp_clip", 0.0)), float(kw.get("dp_noise", 0.0))
        c.dp_clip_quantile, c.dp_clip_lr = float(kw.get("dp_clip_quantile", 0.0)), float(kw.get("dp_clip_lr", 0.2))
        c.dp_count_noise = float(kw.get("dp_count_noise", 0.0))
        assert c.validate() != "", kw


def test_cli_refuses_bad_adaptive_flags():
    from bflc_demo_b200 import run
    from bflc_demo_b200.host import sim
    for argv in (["--dp-clip-quantile", "0.5"], ["--dp-clip", "1", "--dp-clip-quantile", "1.5"],
                 ["--dp-clip", "1", "--dp-clip-quantile", "0.5", "--dp-clip-lr", "-1"],
                 ["--dp-clip", "1", "--dp-noise", "1", "--dp-clip-quantile", "0.5", "--dp-count-noise", "0.4"],
                 ["--dp-clip", "1", "--dp-clip-quantile", "0.5", "--dp-count-noise", "2"]):
        for main in (run.main, sim.main):
            with pytest.raises(SystemExit) as e:
                main(argv)
            assert e.value.code == 2, (main, argv)


def test_host_sim_runs_adaptive_clipping(capsys):
    from bflc_demo_b200.host import sim
    sim.main(["--rounds", "4", "--clients", "10", "--dp-clip", "100", "--dp-clip-quantile", "0.5"])
    out = capsys.readouterr().out
    clips = [float(m) for m in re.findall(r"^clip (\S+) ", out, re.M)]
    assert len(clips) == 4 and clips[0] == 100.0 and clips[-1] < clips[0]      # 100x too large: it falls


def test_nccl_baseline_refuses_adaptive_clipping():
    from bflc_demo_b200.engine.nccl_baseline import NcclBaselineEngine
    with pytest.raises(ValueError, match="differentially private"):
        NcclBaselineEngine(FLConfig.for_world(1, dp_clip=1.0, dp_clip_quantile=0.5), None)


_COMMON = {"flags": 0, "state": 1024, "plan": 2048, "scores": 3072, "meta": 4096, "admit": 5120, "ring": 6144}
# (n_params, ring_slots, extra_bytes, server_state, dp) -> (offsets, total_bytes) of the layouts before adaptive
# clipping existed
PINNED = {
    (4136, 16, 0, 0, False): (dict(_COMMON, work_master=16384, work_shadow=36864, upload_master0=49152,
                                   upload_master1=69632, upload_shadow0=90112, upload_shadow1=102400, **{"global": 114688},
                                   global_shadow=135168, extra=147456), 2097152),
    (4136, 16, 0, 0, True): (dict(_COMMON, work_master=16384, work_shadow=36864, upload_master0=49152,
                                  upload_master1=69632, upload_shadow0=90112, upload_shadow1=102400, **{"global": 114688},
                                  global_shadow=135168, extra=147456, dp=147456), 2097152),
    (11_000_000, 256, 8192, 2, True): (dict(_COMMON, work_master=143360, work_shadow=44146688, upload_master0=66150400,
                                            upload_master1=110153728, upload_shadow0=154157056,
                                            upload_shadow1=176160768, **{"global": 198164480},
                                            global_shadow=242167808, extra=264171520, server_m=264179712,
                                            server_v=308183040, dp=352186368), 352321536),
    (109_483_784, 1024, 0, 1, True): (dict(_COMMON, work_master=548864, work_shadow=438484992, upload_master0=657453056,
                                           upload_master1=1095389184, upload_shadow0=1533325312,
                                           upload_shadow1=1752293376, **{"global": 1971261440},
                                           global_shadow=2409197568, extra=2628165632, server_m=2628165632,
                                           dp=3066101760), 3068133376),
}


@pytest.mark.parametrize("key", list(PINNED))
def test_heap_layout_unchanged_without_adaptive_clipping(key):
    from bflc_demo_b200.parallel.layout import HeapLayout
    P, ring, extra, ss, dp = key
    offsets, total = PINNED[key]
    a = HeapLayout(P, ring, extra_bytes=extra, server_state=ss, dp=dp)
    assert a.offsets == offsets and a.total_bytes == total
    if not dp:
        return
    assert a.dp_region_bytes() == a.sizes["DpPage"] and "dp_bytes" not in a.dp_kwargs(2, 1.0, 1.0, 5)
    c = HeapLayout(P, ring, extra_bytes=extra, server_state=ss, dp=True, dp_adaptive=True)
    assert c.offsets == offsets                               # the adaptive regions grow the last region only
    head, rec = c.dp_adapt_offsets()
    assert head == c.offsets["dp"] + c.sizes["DpPage"] and rec == head + c.sizes["DpAdapt"]
    assert rec + ring * c.sizes["DpClipRecord"] == c.offsets["dp"] + c.dp_region_bytes() <= c.total_bytes
    assert c.dp_kwargs(1, 1.0, 0.0, 5, True)["dp_mode"] == 3 and c.dp_kwargs(2, 1.0, 1.0, 5, True)["dp_mode"] == 4
    assert c.dp_kwargs(2, 1.0, 1.0, 5, True)["dp_bytes"] == c.dp_region_bytes()
    assert a.dp_kwargs(2, 1.0, 1.0, 5, True)["dp_bytes"] == a.sizes["DpPage"]   # too small: the binding refuses it
    assert (c.sizes["DpAdapt"], c.sizes["DpClipRecord"]) == (32, 16)


def test_dp_adapt_header():
    from bflc_demo_b200._native import C
    hdr = np.frombuffer(C().dp_adapt_bytes(2.0, 1.0, 0.5, 0.2, 0.6), F)
    assert hdr[:4].tolist() == [2.0, 0.5, F(0.2), F(0.6)] and hdr[4] == F(privacy.noise_split(1.0, 0.6))


# ------------------------------------------------------------------ ptxas
def test_adaptive_kernels_have_no_stack_frame_or_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("no nvcc")
    inc = [f"-I{build.CSRC / d}" for d in ("include", "ledger", "runtime")]
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, *inc, "-c", str(build.CSRC / "kernels" / "fed_kernels.cu"),
           "-o", str(tmp_path / "f.o")]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    log = proc.stdout + proc.stderr
    assert proc.returncode == 0, log[-3000:]
    props = re.findall(r"Function properties for \w*k_consensus_dp(ILb[01]ELi[0-3]ELi[34]EE)\w*\s*\n\s*"
                       r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    found = {inst: (int(a), int(b), int(c)) for inst, a, b, c in props}
    # adaptive clip under every rule and optimizer, adaptive noise under FedAvg only
    want = {f"ILb{r}ELi{o}ELi{d}EE" for r in (0, 1) for o in range(4) for d in (3, 4) if not (r and d == 4)}
    assert set(found) == want, (sorted(found), log[-3000:])
    assert all(v == (0, 0, 0) for v in found.values()), found
