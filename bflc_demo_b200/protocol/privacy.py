"""Privacy accounting of differentially private aggregation (DP-FedAvg, consensus_math.hpp).

Each noised round releases the FedAvg aggregate of the clipped selected updates plus N(0, sigma^2)
noise per coordinate, sigma = z * C * max_k w_k.  Under replace-one adjacency with fixed weights the
weighted sum's L2 sensitivity is C * max_k w_k, so a round is a Gaussian mechanism with noise
multiplier z, i.e. (1 / z)-GDP, and T rounds compose exactly to mu-GDP with mu = sqrt(T) / z (Dong,
Roth & Su, 2019).  ``epsilon`` converts mu-GDP to (epsilon, delta)-DP exactly; ``rdp_epsilon`` is the
Renyi-DP bound (Mironov, 2017), kept as a cross-check: it is never below ``epsilon``.

What this does NOT cover:
  * the committee's plaintext score rows, the election, and ``n_samples`` / ``avg_cost`` in the block
    record, which are published unprotected;
  * the score-based, data-dependent selection of the updates: the guarantee is about the noised
    combine of the selected set, not about the whole protocol;
  * amplification by subsampling: none is claimed;
  * the floating-point sampler: the accounting assumes an ideal Gaussian, and a floating-point Gaussian
    is not a formally secure sampler (Mironov 2012 shows the attack on floating-point Laplace noise).
"""
from __future__ import annotations

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
