"""Executable specification of the committee-consensus round protocol (pure Python).

This is the oracle every other implementation is diffed against: the C++ ledger runtime
(``csrc/ledger``), the device consensus kernel (``csrc/kernels/fed_kernels.cu``) and the
engines.  It follows SURVEY.md section 1.3, i.e. the behaviour of
``CommitteePrecompiled::call`` (FISCO-BCOS/libprecompiled/extension/CommitteePrecompiled.cpp
:132-456), with the documented decisions:

* true median instead of the reference's order-dependent ``GetMid`` (C:81-115);
* ties broken by ascending client id (reference: unstable sort over hash order, C:365-366);
* a duplicate ``UploadScores`` replaces the row without double counting (C:279-289 bug);
* committee members may not upload updates in their committee round (M:259-263);
* optionally a Byzantine-robust rule (coordinate-wise median or trimmed mean) in place of the
  weighted average of the selected updates (``robust_combine``);
* optionally a server optimizer (FedAvgM momentum, FedAdam, FedYogi) that moves the global model
  along the pseudo-gradient ``global - aggregate`` (``server_step``);
* optionally differentially private aggregation: each selected update clipped to an L2 norm
  (``dp_clip``) and seeded Gaussian noise on the FedAvg aggregate (``dp_gauss``), in the host form of
  ``OracleLedger._aggregate`` and the device form of ``dp_device_combine``.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

EPOCH_NOT_STARTED = -999
ROLE_TRAINER, ROLE_COMM = 1, 2

OK, NOT_STARTED, STALE_EPOCH, DUPLICATE, QUOTA_FULL, NOT_COMMITTEE, UNKNOWN_CLIENT, \
    BAD_PAYLOAD, AGGREGATED, NOT_TRAINER, NOT_READY = range(11)
STATUS_NAMES = ["OK", "NOT_STARTED", "STALE_EPOCH", "DUPLICATE", "QUOTA_FULL", "NOT_COMMITTEE",
                "UNKNOWN_CLIENT", "BAD_PAYLOAD", "AGGREGATED", "NOT_TRAINER", "NOT_READY"]


def true_median(xs: List[float]) -> float:
    s = sorted(np.float32(x) for x in xs)
    n = len(s)
    if n == 0:
        return 0.0
    if n % 2:
        return float(s[n // 2])
    return float(np.float32(0.5) * (s[n // 2 - 1] + s[n // 2]))


AGGREGATIONS = ("fedavg", "median", "trimmed_mean")   # rule id = index (consensus_math.hpp AggRule)


def robust_combine(values, trim: int) -> np.ndarray:
    """Mirror of ``bflc::robust_combine``: coordinate-wise trimmed mean of float32 ``values``
    [n, P], ``min(trim, (n - 1) // 2)`` values dropped at each end (median: any trim >= (n - 1) // 2).
    Values are ordered by the total-order key (NaN canonicalised to 0x7FC00000, then -inf < ... <
    -0 < +0 < ... < +inf < NaN), the kept ones summed left to right in fp32 from -0, and the sum
    divided once by their count."""
    v = np.ascontiguousarray(values, dtype=np.float32)
    n = v.shape[0]
    if n < 1:
        raise ValueError("need at least one value per coordinate")
    b = v.view(np.uint32).copy()
    b[(b & np.uint32(0x7FFFFFFF)) > np.uint32(0x7F800000)] = np.uint32(0x7FC00000)
    neg = (b & np.uint32(0x80000000)) != 0
    key = np.where(neg, ~b, b ^ np.uint32(0x80000000)).astype(np.uint32)
    key.sort(axis=0)
    negk = (key & np.uint32(0x80000000)) == 0
    srt = np.where(negk, ~key, key ^ np.uint32(0x80000000)).astype(np.uint32).view(np.float32)
    t = min(int(trim), (n - 1) // 2)
    s = np.full(v.shape[1:], -0.0, dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(t, n - t):
            s = (s + srt[i]).astype(np.float32)
        return (s / np.float32(n - 2 * t)).astype(np.float32)


def aggregation_trim(aggregation: str, trim: int) -> int:
    """The trim ``robust_combine`` is called with: every value but the middle ones for the median."""
    return 1 << 30 if aggregation == "median" else int(trim)


SERVER_OPTS = ("none", "momentum", "adam", "yogi")   # optimizer id = index (consensus_math.hpp ServerOpt)


def server_constants(lr: float, b1: float, b2: float, tau: float) -> tuple:
    """The six fp32 constants (lr, b1, b2, c1, c2, tau) of ``server_step``: the betas rounded to fp32,
    c1 = fp32(1 - b1) and c2 = fp32(1 - b2) computed in double (``bflc::server_opt_params``)."""
    f = np.float32
    b1, b2 = f(b1), f(b2)
    return (f(lr), b1, b2, f(1.0 - float(b1)), f(1.0 - float(b2)), f(tau))


def server_step(g, a, m, v, opt: str, params):
    """Mirror of ``bflc::server_step`` over float32 arrays: returns (g', m', v') for the global model
    ``g``, the aggregate ``a`` and the state ``m`` / ``v`` (``v`` unused by momentum).  Every operation
    is one correctly rounded fp32 numpy operation, in the order of the C++ definition:
        d = g - a
        momentum: m = b1*m + d;                                   g' = g - lr*m
        adam:     m = b1*m + c1*d; v = b2*v + c2*(d*d);           g' = g - (lr*m) / (sqrt(v) + tau)
        yogi:     m = b1*m + c1*d; v = v - c2*((d*d)*sign(v - d*d)); g' as adam
    ``sign`` is np.sign: +-1, 0 for +-0, NaN for NaN."""
    lr, b1, b2, c1, c2, tau = (np.float32(x) for x in params)
    g, a, m = (np.asarray(x, np.float32) for x in (g, a, m))
    with np.errstate(all="ignore"):
        d = g - a
        if opt == "momentum":
            m = b1 * m + d
            return g - lr * m, m, v
        v = np.asarray(v, np.float32)
        m = b1 * m + c1 * d
        dd = d * d
        if opt == "adam":
            v = b2 * v + c2 * dd
        elif opt == "yogi":
            v = v - c2 * (dd * np.sign(v - dd))
        else:
            raise ValueError(f"unknown server optimizer {opt!r}")
        return g - (lr * m) / (np.sqrt(v) + tau), m, v


# ------------------------------------------------------------------ differential privacy
DP_SITE = 0xD9000000            # consensus_math.hpp kDpSite: Philox counter word 3 of the noise stream
DPSGD_SITE = 0xDA000000         # consensus_math.hpp kDpsgdSite: the same word of DP-SGD's client-side noise
_F = np.float32
_LN2_HI, _LN2_LO = _F(float.fromhex("0x1.62e3p-1")), _F(float.fromhex("0x1.2fefa2p-17"))
_LOG_C = [_F(float.fromhex(h)) for h in ("0x1.c71c72p-4", "0x1.24924ap-3", "0x1.99999ap-3", "0x1.555556p-2")]
_SIN_C = [_F(float.fromhex(h)) for h in ("0x1.71de3ap-19", "-0x1.a01a02p-13", "0x1.111112p-7", "-0x1.555556p-3")]
_COS_C = [_F(float.fromhex(h)) for h in ("-0x1.27e4fcp-22", "0x1.a01a02p-16", "-0x1.6c16c2p-10", "0x1.555556p-5")]
_ANGLE = _F(float.fromhex("0x1.921fb6p-30"))       # pi / 2^31


def dp_mode(clip: float, noise: float) -> int:
    """0 off, 1 clip, 2 clip + noise (consensus_math.hpp dp_mode_of)."""
    return 0 if clip == 0 else 1 if noise == 0 else 2


def philox4x32_10(c, k0: int, k1: int):
    """Philox4x32-10 (philox.hpp) over uint32 counter arrays c = (c0, c1, c2, c3)."""
    M0, M1, W0, W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), 0x9E3779B9, 0xBB67AE85
    c0, c1, c2, c3 = (np.asarray(x, np.uint32) for x in c)
    lo32 = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = c0.astype(np.uint64) * M0
        p1 = c2.astype(np.uint64) * M1
        hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & lo32).astype(np.uint32)
        hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & lo32).astype(np.uint32)
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint32(k0), lo1, hi0 ^ c3 ^ np.uint32(k1), lo0
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return c0, c1, c2, c3


def _dp_log_u(a) -> np.ndarray:
    """Mirror of ``bflc::dp_log_u``: ln((a + 1) / 2^32) from integer operations and fp32 arithmetic."""
    m = np.asarray(a, np.uint32).astype(np.uint64) + np.uint64(1)
    e = (np.frexp(m.astype(np.float64))[1] - 1).astype(np.int64)          # floor(log2 m), exact
    sh = np.maximum(e - 23, 0).astype(np.uint64)
    m_hi = (m >> sh) << sh
    mant = ((m << (63 - e).astype(np.uint64)) >> np.uint64(40)) & np.uint64(0x7FFFFF)
    f = (mant.astype(np.uint32) | np.uint32(0x3F800000)).view(_F)
    c = (m - m_hi).astype(_F) / m_hi.astype(_F)
    big = f.view(np.uint32) > np.uint32(0x3FB504F3)
    f = np.where(big, f * _F(0.5), f).astype(_F)
    e = e + big
    t = (f - _F(1)) / (f + _F(1))
    t2 = t * t
    p = np.full_like(t, _LOG_C[0])
    for k in _LOG_C[1:]:
        p = p * t2 + k
    p = p * t2 + _F(1)
    lf = (t + t) * p + c
    E = (e - 32).astype(_F)
    return (E * _LN2_HI + (E * _LN2_LO + lf)).astype(_F)


def _dp_cossin(k):
    """Mirror of ``bflc::dp_cossin``: (cos, sin) of 2 pi k / 2^32."""
    k = np.asarray(k, np.uint32)
    q = k >> np.uint32(30)
    r = k & np.uint32(0x3FFFFFFF)
    fold = r > np.uint32(0x20000000)
    r = np.where(fold, np.uint32(0x40000000) - r, r).astype(np.uint32)
    x = r.astype(_F) * _ANGLE
    x2 = x * x
    ps = np.full_like(x, _SIN_C[0])
    for k_ in _SIN_C[1:]:
        ps = ps * x2 + k_
    sn = x + (x * x2) * ps
    pc = np.full_like(x, _COS_C[0])
    for k_ in _COS_C[1:]:
        pc = pc * x2 + k_
    pc = pc * x2 + _F(-0.5)
    cs = _F(1) + x2 * pc
    cq, sq = np.where(fold, sn, cs), np.where(fold, cs, sn)
    c = np.select([q == 0, q == 1, q == 2], [cq, -sq, -cq], sq).astype(_F)
    s = np.select([q == 0, q == 1, q == 2], [sq, cq, -sq], -cq).astype(_F)
    return c, s


def dp_box_muller(a, b):
    """Mirror of ``bflc::dp_box_muller`` on uint32 word arrays a (radius) and b (angle)."""
    with np.errstate(all="ignore"):
        lu = _dp_log_u(a)
        r = np.sqrt(_F(0) - (lu + lu)).astype(_F)
        c, s = _dp_cossin(b)
        return (r * c).astype(_F), (r * s).astype(_F)


def dp_gauss(seed: int, epoch: int, first: int, n: int, site: int = DP_SITE) -> np.ndarray:
    """The DP noise xi_i of coordinates first .. first + n - 1 of round ``epoch`` (``bflc::dp_gauss4``):
    coordinate i takes normal i % 4 of Philox call j = i // 4, key = seed, counter = {j_lo, j_hi, epoch,
    site}, normals 0, 1 from output words (x, y) and 2, 3 from (z, w) by Box-Muller.  ``site`` is
    DP_SITE for DP-FedAvg, DPSGD_SITE for DP-SGD (``epoch`` then being the optimizer-step word)."""
    if n <= 0:
        return np.zeros(0, _F)
    j0, j1 = first // 4, (first + n - 1) // 4 + 1
    j = np.arange(j0, j1, dtype=np.uint64)
    w = philox4x32_10(((j & np.uint64(0xFFFFFFFF)).astype(np.uint32), (j >> np.uint64(32)).astype(np.uint32),
                       np.full(j.shape, epoch & 0xFFFFFFFF, np.uint32), np.full(j.shape, site & 0xFFFFFFFF, np.uint32)),
                      seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    z0, z1 = dp_box_muller(w[0], w[1])
    z2, z3 = dp_box_muller(w[2], w[3])
    z = np.stack([z0, z1, z2, z3], axis=1).reshape(-1)
    return z[first - 4 * j0: first - 4 * j0 + n].copy()


def dp_norm(d: np.ndarray) -> np.float32:
    """fp32(sqrt(sum d_i^2)) of float32 ``d``, the exact squares summed in fp64 in ascending index order."""
    d64 = np.asarray(d, _F).astype(np.float64)
    s = np.cumsum(d64 * d64)[-1] if d64.size else 0.0
    with np.errstate(invalid="ignore"):
        return _F(np.sqrt(s))


def dp_scale(norm, clip) -> np.float32:
    """``bflc::dp_scale``: 1 when norm <= clip (compared as bit patterns), else clip / norm in fp32."""
    n, c = _F(norm), _F(clip)
    if np.array(n).view(np.uint32) <= np.array(c).view(np.uint32):
        return _F(1)
    with np.errstate(all="ignore"):
        return _F(c / n)


def dp_clip(g, u, clip, norm=None):
    """One update clipped against the global model ``g``: (v, norm, s), v = u bit for bit when s == 1,
    else g + s * (u - g) in fp32.  ``norm`` (default: ``dp_norm(u - g)``) is the device's when given."""
    g, u = np.asarray(g, _F), np.asarray(u, _F)
    with np.errstate(all="ignore"):
        n = dp_norm((u - g).astype(_F)) if norm is None else _F(norm)
        s = dp_scale(n, clip)
        if np.array(s).view(np.uint32) == np.uint32(0x3F800000):
            return u.copy(), n, s
        return (g + s * (u - g)).astype(_F), n, s


def fmaf(a, b, c) -> np.ndarray:
    """Correctly rounded fp32 fused multiply-add over arrays (the kernel's fmaf): the product is exact
    in fp64, the fp64 sum is rounded to odd, then to fp32 (no double rounding)."""
    a, b, c = (np.asarray(x, _F).astype(np.float64) for x in (a, b, c))
    with np.errstate(all="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        err = (p - (s - bb)) + (c - bb)                     # TwoSum: s + err == p + c exactly
        fix = np.isfinite(s) & np.isfinite(err) & (err != 0)
        bits = s.view(np.uint64).copy()
        away = fix & ((err < 0) != (s < 0))                 # s was rounded away from zero
        bits = np.where(away, bits - np.uint64(1), bits)
        bits = np.where(fix, bits | np.uint64(1), bits)
        return bits.view(np.float64).astype(_F)


def dp_device_combine(g, uploads, weights, norms, rule: str, trim: int, clip: float, noise: float,
                      seed: int, epoch: int) -> np.ndarray:
    """The consensus kernel's DP combine (before any server step): the selected ``uploads`` [K, P] in
    ascending rank order with their consensus ``weights`` and the device's ``norms`` are clipped
    (``dp_clip``), combined by ``rule`` (FedAvg: acc = fmaf(w_k, v_k, acc); otherwise the trimmed mean /
    median of ``robust_combine``), and with ``noise`` > 0 get ``sigma * dp_gauss(seed, epoch, 0, P)``,
    sigma = fp32(fp32(noise * clip) * max_k w_k)."""
    g = np.asarray(g, _F)
    ups = np.asarray(uploads, _F)
    v = np.stack([dp_clip(g, ups[k], clip, norms[k])[0] for k in range(ups.shape[0])])
    if rule == "fedavg":
        acc = np.zeros_like(g)
        for w, x in zip(weights, v):
            acc = fmaf(w, x, acc)
    else:
        acc = robust_combine(v, aggregation_trim(rule, trim))
    if noise > 0:
        sigma = _F(_F(_F(noise) * _F(clip)) * max(_F(w) for w in weights))
        with np.errstate(all="ignore"):
            acc = (acc + sigma * dp_gauss(seed, epoch, 0, g.size)).astype(_F)
    return acc


@dataclass
class ConsensusResult:
    median: Dict[int, float]
    order: List[int]
    selected: List[int]
    weight: Dict[int, float]
    role_after: Dict[int, int]
    global_loss: float


def run_consensus(n: int, n_comm: int, n_aggregate: int, role: Dict[int, int],
                  admitted: List[int], scores: Dict[int, Dict[int, float]],
                  n_samples: Dict[int, int], avg_cost: Dict[int, float],
                  weight_by_score: bool = False) -> ConsensusResult:
    """Mirror of ``bflc::run_consensus`` (csrc/include/consensus_math.hpp)."""
    median: Dict[int, float] = {}
    for t in sorted(admitted):
        col = [scores[c][t] for c in sorted(scores) if (role.get(c, 0) & ROLE_COMM) and t in scores[c]]
        median[t] = true_median(col)
    order = sorted(sorted(admitted), key=lambda t: -median[t])  # stable: ties by ascending id
    k = min(n_aggregate, len(order))
    selected = order[:k]
    w = {}
    for t in selected:
        x = float(n_samples[t])
        if weight_by_score:
            x *= float(np.float32(median[t]))
        w[t] = float(np.float32(x))
    wsum = sum(w.values())
    if k > 0 and wsum <= 0:
        w = {t: 1.0 for t in selected}
        wsum = float(k)
    weight = {t: float(np.float32(w[t] / wsum)) for t in selected}
    cost = np.float32(0)
    for t in selected:
        cost = np.float32(cost + np.float32(avg_cost[t]))
    global_loss = float(cost / np.float32(k)) if k else 0.0
    solo = any((r & ROLE_TRAINER) and (r & ROLE_COMM) for r in role.values())
    role_after = {c: (role[c] if solo else ROLE_TRAINER) for c in role}
    if not solo:
        elected = 0
        for t in order:
            if elected >= n_comm:
                break
            role_after[t] = ROLE_COMM
            elected += 1
        for c in sorted(role):
            if elected >= n_comm:
                break
            if (role[c] & ROLE_COMM) and role_after[c] != ROLE_COMM:
                role_after[c] = ROLE_COMM
                elected += 1
    return ConsensusResult(median, order, sorted(selected), weight, role_after, global_loss)


@dataclass
class OracleLedger:
    client_num: int = 20
    comm_count: int = 4
    aggregate_count: int = 6
    needed_update_count: int = 10
    learning_rate: float = 0.001
    model_size: int = 12
    weight_by_score: bool = False
    solo: bool = False
    aggregation: str = "fedavg"       # fedavg | median | trimmed_mean (of the selected deltas)
    trim: int = 1
    server_opt: str = "none"          # none | momentum | adam | yogi, applied to the aggregate
    server_params: tuple = (1.0, 0.9, 0.99, 0.1, 0.01, 1e-3)   # server_constants(lr, b1, b2, tau)
    dp_clip: float = 0.0              # DP: clip each selected model change lr * delta to this L2 norm (0 = off)
    dp_noise: float = 0.0             # DP: Gaussian noise multiplier on the FedAvg aggregate (0 = clip only)
    dp_seed: int = 0

    epoch: int = EPOCH_NOT_STARTED
    global_model: np.ndarray = field(default=None)
    role: Dict[int, int] = field(default_factory=dict)
    updates: Dict[int, dict] = field(default_factory=dict)
    scores: Dict[int, Dict[int, float]] = field(default_factory=dict)
    arrivals: int = 0
    history: List[dict] = field(default_factory=list)
    server_m: np.ndarray = field(default=None)
    server_v: np.ndarray = field(default=None)

    def __post_init__(self):
        if self.global_model is None:
            self.global_model = np.zeros(self.model_size, dtype=np.float32)
        if self.server_m is None:
            self.server_m = np.zeros(self.model_size, dtype=np.float32)
        if self.server_v is None:
            self.server_v = np.zeros(self.model_size, dtype=np.float32)

    # --- six methods --------------------------------------------------------
    def RegisterNode(self, client: int) -> int:
        if not (0 <= client < self.client_num):
            return UNKNOWN_CLIENT
        if client in self.role:
            return OK
        self.role[client] = ROLE_TRAINER
        if len(self.role) == self.client_num and self.epoch == EPOCH_NOT_STARTED:
            if self.solo:
                for c in self.role:
                    self.role[c] = ROLE_TRAINER | ROLE_COMM
            else:
                for c in sorted(self.role)[: self.comm_count]:
                    self.role[c] = ROLE_COMM
            self.epoch = 0
        return OK

    def QueryState(self, client: int) -> Tuple[int, int]:
        return self.role.get(client, ROLE_TRAINER), self.epoch

    def QueryGlobalModel(self) -> Tuple[np.ndarray, int]:
        return self.global_model.copy(), self.epoch

    def UploadLocalUpdate(self, client: int, delta, n_samples: int, avg_cost: float, ep: int) -> int:
        if self.epoch == EPOCH_NOT_STARTED:
            return NOT_STARTED
        if ep != self.epoch:
            return STALE_EPOCH
        if client not in self.role:
            return UNKNOWN_CLIENT
        if not (self.role[client] & ROLE_TRAINER):
            return NOT_TRAINER
        if client in self.updates:
            return DUPLICATE
        if len(self.updates) >= self.needed_update_count:
            return QUOTA_FULL
        delta = np.asarray(delta, dtype=np.float32)
        if delta.size != self.model_size:
            return BAD_PAYLOAD
        self.updates[client] = dict(delta=delta.copy(), n_samples=int(n_samples),
                                    avg_cost=float(np.float32(avg_cost)), arrival=self.arrivals)
        self.arrivals += 1
        return OK

    def QueryAllUpdates(self) -> List[dict]:
        if len(self.updates) < self.needed_update_count:
            return []
        return [dict(sender=c, **u) for c, u in sorted(self.updates.items(), key=lambda kv: kv[1]["arrival"])]

    def UploadScores(self, client: int, ep: int, scores: Dict[int, float]) -> int:
        if self.epoch == EPOCH_NOT_STARTED:
            return NOT_STARTED
        if ep != self.epoch:
            return STALE_EPOCH
        if not (self.role.get(client, 0) & ROLE_COMM):
            return NOT_COMMITTEE
        if len(self.updates) < self.needed_update_count:
            return NOT_READY
        row = {}
        for t, s in scores.items():
            if t not in self.updates:
                continue
            if not math.isfinite(s):
                return BAD_PAYLOAD
            row[int(t)] = float(np.float32(s))
        self.scores[client] = row
        if len(self.scores) == self.comm_count:
            self._aggregate()
            return AGGREGATED
        return OK

    def _aggregate(self):
        res = run_consensus(self.client_num, self.comm_count, self.aggregate_count, dict(self.role),
                            list(self.updates), self.scores,
                            {c: u["n_samples"] for c, u in self.updates.items()},
                            {c: u["avg_cost"] for c, u in self.updates.items()},
                            self.weight_by_score)
        delta = {t: self.updates[t]["delta"] for t in res.selected}
        dp = dp_mode(self.dp_clip, self.dp_noise)
        if dp:
            # the model change is lr * delta; a clipped update enters the rule as s * delta
            lr = np.float32(self.learning_rate)
            for t in res.selected:
                with np.errstate(all="ignore"):
                    s = dp_scale(dp_norm((lr * delta[t]).astype(np.float32)), self.dp_clip)
                    if np.array(s).view(np.uint32) != np.uint32(0x3F800000):
                        delta[t] = (s * delta[t]).astype(np.float32)
        total = np.zeros(self.model_size, dtype=np.float32)
        if self.aggregation == "fedavg":
            for t in sorted(res.selected):
                total = (np.float32(res.weight[t]) * delta[t] + total).astype(np.float32)
        elif res.selected:
            total = robust_combine(np.stack([delta[t] for t in sorted(res.selected)]),
                                   aggregation_trim(self.aggregation, self.trim))
        agg = (self.global_model - np.float32(self.learning_rate) * total).astype(np.float32)
        if dp == 2 and res.selected:
            sigma = np.float32(np.float32(np.float32(self.dp_noise) * np.float32(self.dp_clip))
                               * max(np.float32(res.weight[t]) for t in res.selected))
            with np.errstate(all="ignore"):
                agg = (agg + sigma * dp_gauss(self.dp_seed, self.epoch, 0, self.model_size)).astype(np.float32)
        if self.server_opt == "none":
            self.global_model = agg
        elif res.selected:                  # a round without a selection leaves model and state alone
            self.global_model, self.server_m, self.server_v = server_step(
                self.global_model, agg, self.server_m, self.server_v, self.server_opt, self.server_params)
        self.history.append(dict(epoch=self.epoch, selected=res.selected, weight=res.weight,
                                 median=res.median, role_after=dict(res.role_after),
                                 global_loss=res.global_loss, order=res.order))
        self.role = dict(res.role_after)
        self.updates = {}
        self.scores = {}
        self.epoch += 1
