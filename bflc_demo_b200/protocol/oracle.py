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
  along the pseudo-gradient ``global - aggregate`` (``server_step``).
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
        total = np.zeros(self.model_size, dtype=np.float32)
        if self.aggregation == "fedavg":
            for t in sorted(res.selected):
                total = (np.float32(res.weight[t]) * self.updates[t]["delta"] + total).astype(np.float32)
        elif res.selected:
            total = robust_combine(np.stack([self.updates[t]["delta"] for t in sorted(res.selected)]),
                                   aggregation_trim(self.aggregation, self.trim))
        agg = (self.global_model - np.float32(self.learning_rate) * total).astype(np.float32)
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
