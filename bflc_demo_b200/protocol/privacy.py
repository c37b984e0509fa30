"""Privacy accounting of differentially private aggregation (DP-FedAvg, consensus_math.hpp).

Each noised round releases the FedAvg aggregate of the clipped selected updates plus N(0, sigma^2)
noise per coordinate, sigma = z * C * max_k w_k.  Under add/remove-one adjacency (one selected update
present or absent) with fixed weights the weighted sum's L2 sensitivity is C * max_k w_k, so a round is
a Gaussian mechanism with noise multiplier z, i.e. (1 / z)-GDP, and T rounds compose exactly to mu-GDP
with mu = sqrt(T) / z (Dong, Roth & Su, 2019).  (Under replace-one adjacency the sensitivity is
2 C max_k w_k; that is not the convention accounted here.)  ``epsilon`` converts mu-GDP to
(epsilon, delta)-DP exactly; ``rdp_epsilon`` is the Renyi-DP bound (Mironov, 2017), kept as a
cross-check: it is never below ``epsilon``.

With adaptive clipping the clipped count's centred bits b - n_sel / 2 move by 1/2 under the same
adjacency; the count gets noise sigma_b and the aggregate z_delta (``noise_split``), which together are
one Gaussian mechanism with multiplier z (Andrew et al. 2021, Theorem 1), so ``epsilon`` is unchanged for
the same (z, T, delta).

DP-SGD with Poisson sampling (``FLConfig.dpsgd_sampling = "poisson"``) is accounted with the Renyi DP of the
sampled Gaussian mechanism (Mironov, Talwar & Zhang, 2019), ``sampled_gaussian_rdp``, composed over the steps and
converted to (epsilon, delta) by Balle et al. 2020, Thm 21 (``poisson_epsilon``).  ``poisson_capacity`` sizes the
fixed-capacity batch the device sampler fills; its tail ``binomial_tail`` is the truncation term of the delta.

What this does NOT cover:
  * the committee's plaintext score rows, the election, and ``n_samples`` / ``avg_cost`` in the block
    record, which are published unprotected;
  * the score-based, data-dependent selection of the updates: the guarantee is about the noised
    combine of the selected set, not about the whole protocol;
  * amplification by subsampling for DP-FedAvg or for partition-sampled DP-SGD: none is claimed;
  * the floating-point sampler: the accounting assumes an ideal Gaussian, and a floating-point Gaussian
    is not a formally secure sampler (Mironov 2012 shows the attack on floating-point Laplace noise).
"""
from __future__ import annotations

import functools
import math

_SQRT2 = math.sqrt(2.0)


def _log_phi(x: float) -> float:
    """log Phi(x), accurate far into the lower tail (x << 0) where Phi underflows."""
    if x > -30.0:
        return math.log(0.5 * math.erfc(-x / _SQRT2))
    # Phi(x) = phi(x) / |x| * (1 - 1/x^2 + 3/x^4 - 15/x^6 + ...), |x| >= 30: the series' error < 1e-12
    y = -x
    s = 1.0 - 1.0 / y ** 2 + 3.0 / y ** 4 - 15.0 / y ** 6 + 105.0 / y ** 8
    return -0.5 * y * y - math.log(y) - 0.5 * math.log(2.0 * math.pi) + math.log(s)


def gdp_mu(z: float, rounds: int) -> float:
    """mu of ``rounds`` composed Gaussian mechanisms with noise multiplier ``z``."""
    if not (z > 0 and math.isfinite(z)):
        raise ValueError("noise multiplier z must be finite and > 0")
    if rounds < 0:
        raise ValueError("rounds must be >= 0")
    return math.sqrt(rounds) / z


def gdp_delta(eps: float, mu: float) -> float:
    """delta(eps) of mu-GDP: Phi(-eps/mu + mu/2) - e^eps Phi(-eps/mu - mu/2), the second term in log space
    so a large eps does not overflow."""
    a = -eps / mu + mu / 2.0
    b = -eps / mu - mu / 2.0
    return math.exp(_log_phi(a)) - math.exp(eps + _log_phi(b))


def epsilon(z: float, rounds: int, delta: float) -> float:
    """The smallest eps such that ``rounds`` noised rounds with noise multiplier ``z`` are
    (eps, delta)-DP: the root of gdp_delta(eps, sqrt(rounds) / z) = delta, by bisection."""
    if not 0 < delta < 1:
        raise ValueError("delta must lie in (0, 1)")
    mu = gdp_mu(z, rounds)
    if mu == 0 or gdp_delta(0.0, mu) <= delta:
        return 0.0
    lo, hi = 0.0, 1.0
    while gdp_delta(hi, mu) > delta:       # delta(eps) decreases in eps
        lo, hi = hi, 2.0 * hi
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        if gdp_delta(mid, mu) > delta:
            lo = mid
        else:
            hi = mid
        if hi - lo <= 1e-13 * hi:
            break
    return hi


def rdp_epsilon(z: float, rounds: int, delta: float) -> float:
    """Renyi-DP bound: the Gaussian mechanism is (alpha, alpha / (2 z^2))-RDP, T rounds compose to
    alpha T / (2 z^2), and eps = min over alpha > 1 of alpha T / (2 z^2) + log(1/delta) / (alpha - 1)
    = A + 2 sqrt(A B) with A = T / (2 z^2), B = log(1 / delta)."""
    if not 0 < delta < 1:
        raise ValueError("delta must lie in (0, 1)")
    gdp_mu(z, rounds)
    a = rounds / (2.0 * z * z)
    if a == 0:
        return 0.0
    b = math.log(1.0 / delta)
    return a + 2.0 * math.sqrt(a * b)


# ------------------------------------------------------------------ Poisson-sampled DP-SGD
POISSON_ETA = 2.0 ** -40          # the largest overflow probability per step a batch capacity may leave
RDP_ORDERS = tuple(range(2, 257))  # the integer Renyi orders epsilon is minimised over


def _logsumexp(v) -> float:
    m = max(v)
    if m == -math.inf:
        return -math.inf
    return m + math.log(math.fsum(math.exp(x - m) for x in v))


def sampled_gaussian_rdp(q: float, z: float, alpha: int) -> float:
    """Renyi DP of order ``alpha`` (an integer >= 2) of one step of the sampled Gaussian mechanism with sampling
    rate q and noise multiplier z: log sum_{k=0}^{alpha} C(alpha, k) (1 - q)^(alpha - k) q^k exp((k^2 - k) /
    (2 z^2)) / (alpha - 1), in log space (Mironov, Talwar & Zhang 2019, Sec. 3.3, integer alpha)."""
    alpha = int(alpha)
    if alpha < 2:
        raise ValueError("alpha must be an integer >= 2")
    if not 0 < q <= 1:
        raise ValueError("q must lie in (0, 1]")
    if not (z > 0 and math.isfinite(z)):
        raise ValueError("noise multiplier z must be finite and > 0")
    if q == 1:
        return alpha / (2.0 * z * z)
    lq, l1q = math.log(q), math.log1p(-q)
    terms = [math.lgamma(alpha + 1) - math.lgamma(k + 1) - math.lgamma(alpha - k + 1) + (alpha - k) * l1q + k * lq
             + (k * k - k) / (2.0 * z * z) for k in range(alpha + 1)]
    return _logsumexp(terms) / (alpha - 1)


def rdp_to_epsilon(rdp: float, alpha: int, delta: float) -> float:
    """(alpha, rdp)-RDP -> (eps, delta)-DP, Balle et al. 2020 Thm 21: rdp + log((alpha - 1) / alpha) - (log delta +
    log alpha) / (alpha - 1), floored at 0."""
    eps = rdp + math.log((alpha - 1) / alpha) - (math.log(delta) + math.log(alpha)) / (alpha - 1)
    return max(eps, 0.0)


def poisson_epsilon(q: float, z: float, steps: int, delta: float) -> float:
    """epsilon of ``steps`` composed sampled Gaussian steps (rate q, noise multiplier z) at ``delta``: the
    minimum over the integer orders 2 .. 256 of ``rdp_to_epsilon(steps * sampled_gaussian_rdp)``.  0 for no
    steps, inf without noise."""
    if not 0 < delta < 1:
        raise ValueError("delta must lie in (0, 1)")
    if steps < 0:
        raise ValueError("steps must be >= 0")
    if steps == 0:
        return 0.0
    if z == 0:
        return math.inf
    return min(rdp_to_epsilon(steps * sampled_gaussian_rdp(q, z, a), a, delta) for a in RDP_ORDERS)


def _log_pmf(n: int, q: float, j: int, c: float, lq: float, l1q: float) -> float:
    return c - math.lgamma(j + 1) - math.lgamma(n - j + 1) + j * lq + ((n - j) * l1q if n > j else 0.0)


_TAIL_REL = -80.0      # stop a sum once the whole rest of it is below e^-80 of what is summed


def binomial_log_tail(n: int, q: float, k: int) -> float:
    """log P[Binomial(n, q) > k] in log space (the pmf from lgamma, summed with logsumexp); -inf for k >= n.

    Only the terms that matter are summed.  Past the mode the pmf ratio r_j = (n - j) q / ((j + 1) (1 - q)) is
    below 1 and falls with j, so the rest of the sum after term j is at most pmf_j r_j / (1 - r_j): the upper
    tail stops once that bound is below e^-80 of the partial sum.  For k below the mode the tail is 1 minus the
    lower sum P[X <= k], summed downwards from k with the same bound on the ratios' inverses."""
    if k >= n:
        return -math.inf
    if k < 0:
        return 0.0
    if q >= 1:
        return 0.0
    lq, l1q, c = math.log(q), math.log1p(-q), math.lgamma(n + 1)
    mode = math.floor((n + 1) * q)
    if k + 1 >= mode:              # upper tail, terms falling from j = k + 1
        terms, j = [], k + 1
        while j <= n:
            t = _log_pmf(n, q, j, c, lq, l1q)
            terms.append(t)
            r = (n - j) * q / ((j + 1) * (1 - q))
            if r <= 0 or (r < 1 and t + math.log(r / (1 - r)) < _logsumexp(terms) + _TAIL_REL):
                break
            j += 1
        return _logsumexp(terms)
    # below the mode: 1 - P[X <= k], terms falling from j = k downwards
    terms, j = [], k
    while j >= 0:
        t = _log_pmf(n, q, j, c, lq, l1q)
        terms.append(t)
        r = j * (1 - q) / ((n - j + 1) * q)        # pmf_{j-1} / pmf_j
        if r <= 0 or (r < 1 and t + math.log(r / (1 - r)) < _logsumexp(terms) + _TAIL_REL):
            break
        j -= 1
    return math.log1p(-min(math.exp(_logsumexp(terms)), 1.0))


def binomial_tail(n: int, q: float, k: int) -> float:
    """P[Binomial(n, q) > k]."""
    return math.exp(binomial_log_tail(n, q, k))


@functools.lru_cache(maxsize=64)
def poisson_capacity(S: int, q: float) -> int:
    """The batch capacity of Poisson sampling at rate q over S records: the smallest multiple of 8 k with
    P[Binomial(S, q) > k] <= POISSON_ETA, and at most S (where no overflow can happen)."""
    if S < 1 or not 0 < q <= 1:
        raise ValueError("poisson_capacity needs S >= 1 and q in (0, 1]")
    log_eta = math.log(POISSON_ETA)
    lo, hi = 0, (S + 7) // 8       # in units of 8: the tail falls as k grows, so bisect
    while lo < hi:
        mid = (lo + hi) // 2
        if binomial_log_tail(S, q, 8 * mid) <= log_eta:
            hi = mid
        else:
            lo = mid + 1
    return min(8 * lo, S)


def noise_split(z: float, count_noise: float) -> float:
    """Adaptive clipping's split of the total noise multiplier ``z`` (Andrew et al. 2021, Theorem 1): the
    aggregate's multiplier z_delta = (z^-2 - (2 sigma_b)^-2)^-1/2 when the clipped count carries noise
    sigma_b > z / 2 (so that (2 sigma_b)^-2 < z^-2).  One round is then the Gaussian mechanism with multiplier z, so ``epsilon`` is that
    of DP-FedAvg at z.  Computed in double from the fp32 inputs and rounded to fp32, exactly as
    ``bflc::dp_noise_split`` (the kernel, the ledger and the oracle use this value)."""
    import numpy as np
    z, sb = float(np.float32(z)), float(np.float32(count_noise))
    if not 2.0 * sb > z:
        raise ValueError("count_noise must exceed z / 2")
    a = 1.0 / (z * z)
    s2 = 2.0 * sb
    return float(np.float32(1.0 / math.sqrt(a - 1.0 / (s2 * s2))))
