// The committee-consensus decision procedure, written once and compiled for both the
// host C++ ledger and the device consensus kernel, so the HBM ledger replicas and the
// host chain can never disagree on an election.
//
// Spec = reference `CommitteePrecompiled::Aggregate`
// (FISCO-BCOS/libprecompiled/extension/CommitteePrecompiled.cpp:349-456):
//   0. per-trainer score = median over the committee's scores          (C:351-362)
//   1. rank trainers by score, descending                               (C:365-366)
//   2-3. aggregate the top AGGREGATE_COUNT, weighted by n_samples       (C:373-400)
//   5. next committee = top COMM_COUNT scorers; old committee -> trainer (C:444-455)
// Deliberate deviations (SURVEY.md 1.3 / 7.1):
//   * true median (mean of the two middle values for even counts); the reference's
//     quickselect `GetMid` (C:81-115) is input-order dependent and is NOT emulated;
//   * ties are broken by ascending rank id (the reference: unstable sort over
//     unordered_map order);
//   * optional score-weighted aggregation (`weight_by_score`), default off = reference;
//   * optional Byzantine-robust aggregation of the selected updates (coordinate-wise median or
//     trimmed mean, robust_combine), default off = FedAvg;
//   * optional server optimizer on the aggregate (FedAvgM momentum, FedAdam, FedYogi,
//     server_step), default off = the aggregate is the new global model;
//   * optional differentially private aggregation (DP-FedAvg: per-update L2 clipping, dp_scale,
//     and seeded Gaussian noise on the aggregate, dp_gauss4), default off.
#pragma once
#include <cmath>
#include <cstdint>

#include "philox.hpp"

#if defined(__CUDACC__)
#define BFLC_HD __host__ __device__ __forceinline__
#define BFLC_UNROLL _Pragma("unroll")
#else
#define BFLC_HD inline
#define BFLC_UNROLL
#endif

namespace bflc {

constexpr int kCMaxRanks = 64;  // host ledger supports up to 64 clients; device path uses <= 8

enum RoleBits : uint32_t { ROLE_TRAINER = 1u, ROLE_COMM = 2u };

template <int MAXR>
struct ConsensusIn {
  int n_ranks;
  int n_comm;        // COMM_COUNT
  int n_aggregate;   // AGGREGATE_COUNT
  int weight_by_score;
  uint32_t role[MAXR];          // RoleBits
  uint8_t admitted[MAXR];       // 1 = this rank's update was admitted this round
  uint8_t scored[MAXR][MAXR];   // scored[c][t] = committee c supplied a score for trainer t
  float score[MAXR][MAXR];      // score[c][t]
  uint32_t n_samples[MAXR];
  float avg_cost[MAXR];
};

template <int MAXR>
struct ConsensusOut {
  float median[MAXR];
  int order[MAXR];      // admitted trainers sorted by (median desc, rank asc)
  int n_ranked;
  int n_selected;
  uint8_t selected[MAXR];
  float weight[MAXR];   // aggregation weights, sum to 1 over the selected trainers
  uint32_t role_after[MAXR];
  float global_loss;
};

// Median of the n scores in v[MAXR] (the other slots hold +inf; scores are finite), the values
// at the middle positions of a stable ascending sort.  Each value's position is counted, not
// found by sorting in place, so the device keeps v in registers (no local-memory stack frame).
template <int MAXR>
BFLC_HD float median_of(const float* v, int n) {
  float lo = 0.f, hi = 0.f;
BFLC_UNROLL
  for (int i = 0; i < MAXR; ++i) {
    int r = 0;
BFLC_UNROLL
    for (int j = 0; j < MAXR; ++j) r += (v[j] < v[i] || (j < i && v[j] == v[i])) ? 1 : 0;
    lo = r == (n - 1) / 2 ? v[i] : lo;
    hi = r == n / 2 ? v[i] : hi;
  }
  if (n <= 0) return 0.f;
  return (n & 1) ? hi : 0.5f * (lo + hi);
}

// ---------------------------------------------------------------- robust aggregation
// Byzantine-robust rules applied per coordinate to the selected updates (after the score
// filter).  FedAvg stays the sample-weighted sum in the callers; the two robust rules share ONE
// code path: median is the trimmed mean at the largest trim, (n - 1) / 2.
enum AggRule : int { AGG_FEDAVG = 0, AGG_MEDIAN = 1, AGG_TRIMMED_MEAN = 2 };
constexpr int kMaxTrim = 255;  // the trim travels in 8 bits of the device block record

BFLC_HD bool agg_rule_valid(int rule, int trim) {
  return rule == AGG_FEDAVG || rule == AGG_MEDIAN || (rule == AGG_TRIMMED_MEAN && trim >= 1 && trim <= kMaxTrim);
}
// The record / snapshot word of a rule: rule | trim << 8, the trim kept only where it matters.  The
// block record's word also carries the server optimizer (ServerOpt below) in bits 16..23 and the DP
// mode (DpMode below) in bit 24 (clip) and bit 25 (noise); "none" and "off" leave every word
// unchanged.
BFLC_HD uint32_t agg_word(int rule, int trim, int server_opt = 0, int dp = 0) {
  return static_cast<uint32_t>(rule) | (rule == AGG_TRIMMED_MEAN ? static_cast<uint32_t>(trim) << 8 : 0u) |
         static_cast<uint32_t>(server_opt) << 16 | (dp >= 1 ? 1u << 24 : 0u) | (dp >= 2 ? 1u << 25 : 0u);
}
// Values dropped at each end for n selected updates.
BFLC_HD int agg_trim(int rule, int trim, int n) {
  const int half = n > 0 ? (n - 1) / 2 : 0;
  return rule == AGG_MEDIAN ? half : (trim < half ? trim : half);
}

// Total order over fp32 bit patterns: -inf < ... < -0 < +0 < ... < +inf < NaN, every NaN first
// canonicalised to 0x7FC00000, so the sorted sequence (and with it the result) is unique.
BFLC_HD uint32_t agg_key(float v) {
#if defined(__CUDA_ARCH__)
  uint32_t b = __float_as_uint(v);
#else
  uint32_t b;
  __builtin_memcpy(&b, &v, 4);
#endif
  b = (b & 0x7FFFFFFFu) > 0x7F800000u ? 0x7FC00000u : b;
  return (b & 0x80000000u) ? ~b : (b ^ 0x80000000u);
}
BFLC_HD float agg_key_value(uint32_t k) {
  const uint32_t b = (k & 0x80000000u) ? (k ^ 0x80000000u) : ~k;
#if defined(__CUDA_ARCH__)
  return __uint_as_float(b);
#else
  float v;
  __builtin_memcpy(&v, &b, 4);
  return v;
#endif
}

// Trimmed mean of v[0..n), t values dropped at each end (0 <= t <= (n - 1) / 2, 1 <= n <= MAXR):
// odd-even transposition sort over the keys (n phases; slots >= n hold the largest key and never
// move), then a left-to-right fp32 sum of the kept values and one correctly rounded division.
// Fully unrolled over MAXR, so on the device every value stays in a register.
template <int MAXR>
BFLC_HD float robust_combine(const float* v, int n, int t) {
  uint32_t k[MAXR];
BFLC_UNROLL
  for (int i = 0; i < MAXR; ++i) k[i] = i < n ? agg_key(v[i]) : 0xFFFFFFFFu;
BFLC_UNROLL
  for (int p = 0; p < MAXR; ++p) {
    if (p < n) {
BFLC_UNROLL
      for (int i = p & 1; i + 1 < MAXR; i += 2) {
        const uint32_t a = k[i], b = k[i + 1];
        k[i] = a < b ? a : b;
        k[i + 1] = a < b ? b : a;
      }
    }
  }
  float s = -0.0f;  // the additive identity for every value, -0 included
BFLC_UNROLL
  for (int i = 0; i < MAXR; ++i) {
    if (i >= t && i < n - t) {
#if defined(__CUDA_ARCH__)
      s = __fadd_rn(s, agg_key_value(k[i]));
#else
      s = s + agg_key_value(k[i]);
#endif
    }
  }
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(s, static_cast<float>(n - 2 * t));
#else
  return s / static_cast<float>(n - 2 * t);
#endif
}

// ---------------------------------------------------------------- server optimizer
// Applied per coordinate to the aggregate a (what the rule above produced) and the current global
// model g, along the pseudo-gradient d = g - a (FedAvgM, Hsu et al. 2019; FedAdam / FedYogi, Reddi
// et al. 2021, without bias correction, m = v = 0 at genesis):
//   momentum: m = b1*m + d;                                        g' = g - lr*m
//   adam:     m = b1*m + c1*d; v = b2*v + c2*(d*d);                g' = g - (lr*m) / (sqrt(v) + tau)
//   yogi:     m = b1*m + c1*d; v = v - c2*((d*d)*sign(v - d*d));   g' as adam
// The callers skip it for a round that selects nothing (model and state stay as they are).
enum ServerOpt : int { SOPT_NONE = 0, SOPT_MOMENTUM = 1, SOPT_ADAM = 2, SOPT_YOGI = 3 };

// The six fp32 constants every implementation uses; c1 = fp32(1 - b1) and c2 = fp32(1 - b2) are
// computed once, in double from the fp32 betas (server_opt_params), never inside a step.
struct ServerOptParams {
  float lr, b1, b2, c1, c2, tau;
};
inline ServerOptParams server_opt_params(float lr, float b1, float b2, float tau) {
  return ServerOptParams{lr, b1, b2, static_cast<float>(1.0 - static_cast<double>(b1)),
                         static_cast<float>(1.0 - static_cast<double>(b2)), tau};
}
// "" when the optimizer id and its hyperparameters are usable: lr > 0 finite, 0 <= b1 < 1, and for
// adam / yogi 0 <= b2 < 1 and tau > 0 finite
inline const char* server_opt_check(int opt, float lr, float b1, float b2, float tau) {
  if (opt < SOPT_NONE || opt > SOPT_YOGI) return "server_opt must be 0 (none), 1 (momentum), 2 (adam) or 3 (yogi)";
  if (opt == SOPT_NONE) return "";
  if (!(std::isfinite(lr) && lr > 0.f)) return "server_lr must be finite and > 0";
  if (!(b1 >= 0.f && b1 < 1.f)) return "server_beta1 must lie in [0, 1)";
  if (opt == SOPT_MOMENTUM) return "";
  if (!(b2 >= 0.f && b2 < 1.f)) return "server_beta2 must lie in [0, 1)";
  if (!(std::isfinite(tau) && tau > 0.f)) return "server_tau must be finite and > 0";
  return "";
}
// fp32 vectors of optimizer state: m for momentum, m and v for adam / yogi
BFLC_HD int server_state_vectors(int opt) { return opt == SOPT_NONE ? 0 : opt == SOPT_MOMENTUM ? 1 : 2; }

// One correctly rounded fp32 operation each, never contracted into an FMA.  On the device these are
// the IEEE PTX instructions without .ftz: the build's --use_fast_math would turn __fadd_rn & co.
// into their flush-to-zero forms, and the state must evolve exactly as on the host (subnormals
// included).
#if defined(__CUDA_ARCH__)
#define BFLC_SOP2(name, ins)                                                 \
  __device__ __forceinline__ float name(float a, float b) {                  \
    float r;                                                                 \
    asm(ins " %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));                      \
    return r;                                                                \
  }
BFLC_SOP2(so_add, "add.rn.f32")
BFLC_SOP2(so_sub, "sub.rn.f32")
BFLC_SOP2(so_mul, "mul.rn.f32")
BFLC_SOP2(so_div, "div.rn.f32")
#undef BFLC_SOP2
__device__ __forceinline__ float so_sqrt(float a) {
  float r;
  asm("sqrt.rn.f32 %0, %1;" : "=f"(r) : "f"(a));
  return r;
}
#else
inline float so_add(float a, float b) { return a + b; }
inline float so_sub(float a, float b) { return a - b; }
inline float so_mul(float a, float b) { return a * b; }
inline float so_div(float a, float b) { return a / b; }
inline float so_sqrt(float a) { return std::sqrt(a); }
#endif
// np.sign: +1, -1, +0 for either zero, NaN for NaN (a (x > 0) - (x < 0) would give 0 for NaN).
// Decided from the bit pattern: float compares compile to setp.*.ftz under --use_fast_math and
// would call a subnormal v - d*d zero on the device.
BFLC_HD float so_sign(float x) {
#if defined(__CUDA_ARCH__)
  const uint32_t b = __float_as_uint(x);
#else
  uint32_t b;
  __builtin_memcpy(&b, &x, 4);
#endif
  if ((b & 0x7FFFFFFFu) > 0x7F800000u) return x;   // NaN
  if ((b & 0x7FFFFFFFu) == 0u) return 0.f;         // +-0
  return (b & 0x80000000u) ? -1.f : 1.f;
}

// One coordinate: returns g', updates m (and v for adam / yogi).  opt is a compile-time constant in
// the kernel, so only its own branch is emitted there.
BFLC_HD float server_step(int opt, float g, float a, float& m, float& v, const ServerOptParams& p) {
  const float d = so_sub(g, a);
  if (opt == SOPT_MOMENTUM) {
    m = so_add(so_mul(p.b1, m), d);
    return so_sub(g, so_mul(p.lr, m));
  }
  m = so_add(so_mul(p.b1, m), so_mul(p.c1, d));
  const float dd = so_mul(d, d);
  if (opt == SOPT_ADAM)
    v = so_add(so_mul(p.b2, v), so_mul(p.c2, dd));
  else
    v = so_sub(v, so_mul(p.c2, so_mul(dd, so_sign(so_sub(v, dd)))));
  return so_sub(g, so_div(so_mul(p.lr, m), so_add(so_sqrt(v), p.tau)));
}

// ---------------------------------------------------------------- differential privacy
// DP-FedAvg (McMahan et al. 2018) on the selected uploads u_k and the current global model g:
//   n_k = fp32(sqrt(sum_i d_i * d_i)), d_i = u_k,i - g_i in fp32, d_i * d_i exact in fp64, summed in fp64
//   s_k = 1 if n_k <= C else C / n_k;  v_k = u_k if s_k == 1 else g + s_k * (u_k - g)
//   the configured rule combines the v_k; with noise (FedAvg only) coordinate i of the aggregate gets
//   sigma * xi_i, sigma = (z * C) * max_k w_k, xi_i = dp_gauss4(seed, epoch, i / 4)[i % 4]
// The host ledger applies the same definition to its delta form, where the model change is lr * delta
// (see Ledger::aggregate_locked).  Floating-point Gaussian noise is not a formally secure sampler
// (Mironov 2012); the mechanism's guarantee is stated for an ideal Gaussian (DESIGN.md).
enum DpMode : int { DP_OFF = 0, DP_CLIP = 1, DP_NOISE = 2 };
// Philox counter word 3 of the noise stream: above every dropout site (< 2^24, philox.hpp), and the
// key is the DP seed, not a dropout seed
constexpr uint32_t kDpSite = 0xD9000000u;
// Counter word 3 of DP-SGD's client-side noise (dpsgd_kernels.cu): apart from kDpSite and above every
// dropout site, so no stream of one mechanism ever repeats a stream of another, whatever the keys
constexpr uint32_t kDpsgdSite = 0xDA000000u;

// "" when the mode and its parameters are usable: clip > 0 finite for clip and noise, noise > 0
// finite only with noise, which needs the FedAvg rule (the L2 sensitivity of a median or a trimmed
// mean is not bounded by the clip)
inline const char* dp_check(int mode, float clip, float noise, int rule) {
  if (mode < DP_OFF || mode > DP_NOISE) return "dp mode must be 0 (off), 1 (clip) or 2 (clip + noise)";
  if (mode == DP_OFF) return (clip == 0.f && noise == 0.f) ? "" : "dp_clip and dp_noise must be 0 with DP off";
  if (!(std::isfinite(clip) && clip > 0.f)) return "dp_clip must be finite and > 0";
  if (mode == DP_CLIP) return noise == 0.f ? "" : "dp_noise must be 0 for clipping without noise";
  if (!(std::isfinite(noise) && noise > 0.f)) return "dp_noise must be finite and > 0";
  if (rule != AGG_FEDAVG) return "dp_noise needs the FedAvg rule";
  return "";
}
// the mode of a (clip, noise) pair: 0 off, 1 clip, 2 clip + noise
inline int dp_mode_of(float clip, float noise) { return clip == 0.f ? DP_OFF : noise == 0.f ? DP_CLIP : DP_NOISE; }

BFLC_HD uint32_t dp_bits(float x) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(x);
#else
  uint32_t b;
  __builtin_memcpy(&b, &x, 4);
  return b;
#endif
}
BFLC_HD float dp_float(uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __uint_as_float(b);
#else
  float x;
  __builtin_memcpy(&x, &b, 4);
  return x;
#endif
}
// fp32 of the square root of an fp64 sum of squares (each rounding correctly rounded, IEEE)
BFLC_HD float dp_norm(double sumsq) {
#if defined(__CUDA_ARCH__)
  return __double2float_rn(__dsqrt_rn(sumsq));
#else
  return static_cast<float>(std::sqrt(sumsq));
#endif
}
// The clip factor.  n >= +0 or NaN and C > 0 finite, so n <= C is an unsigned compare of the bit
// patterns (a float compare would flush subnormals under --use_fast_math); a NaN norm gives NaN.
BFLC_HD float dp_scale(float n, float clip) { return dp_bits(n) <= dp_bits(clip) ? 1.f : so_div(clip, n); }
// One clipped coordinate: g + s * (u - g)
BFLC_HD float dp_clip_value(float g, float u, float s) { return so_add(g, so_mul(s, so_sub(u, g))); }

// ln(u), u = (a + 1) / 2^32 in [2^-32, 1]: m = a + 1 = 2^e * f * (1 + rem / m_hi) with f in [1, 2) the
// top 24 bits of m (exact), rem the bits below them; f > sqrt(2) is halved (exact) so that
// ln f = 2 atanh(t), t = (f - 1) / (f + 1), |t| < 0.172, is a short odd series; ln(1 + rem / m_hi)
// (< 2^-23) is its first-order term.  ln u = (e - 32) ln 2 + ln f + rem / m_hi, ln 2 split so that
// (e - 32) * ln2_hi is exact.
BFLC_HD float dp_log_u(uint32_t a) {
  const uint64_t m = static_cast<uint64_t>(a) + 1u;
#if defined(__CUDA_ARCH__)
  int e = 63 - __clzll(static_cast<long long>(m));
#else
  int e = 63 - __builtin_clzll(m);
#endif
  const int sh = e > 23 ? e - 23 : 0;
  const uint64_t m_hi = (m >> sh) << sh;
  const uint32_t mant = static_cast<uint32_t>((m << (63 - e)) >> 40) & 0x7FFFFFu;
  float f = dp_float(0x3F800000u | mant);
  const float c = so_div(static_cast<float>(static_cast<uint32_t>(m - m_hi)), static_cast<float>(m_hi));
  if (dp_bits(f) > 0x3FB504F3u) {   // f > fp32(sqrt(2))
    f = so_mul(f, 0.5f);
    ++e;
  }
  const float t = so_div(so_sub(f, 1.f), so_add(f, 1.f));
  const float t2 = so_mul(t, t);
  float p = 0x1.c71c72p-4f;                        // 1/9
  p = so_add(so_mul(p, t2), 0x1.24924ap-3f);       // 1/7
  p = so_add(so_mul(p, t2), 0x1.99999ap-3f);       // 1/5
  p = so_add(so_mul(p, t2), 0x1.555556p-2f);       // 1/3
  p = so_add(so_mul(p, t2), 1.f);
  const float lf = so_add(so_mul(so_add(t, t), p), c);
  const float E = static_cast<float>(e - 32);
  return so_add(so_mul(E, 0x1.62e3p-1f), so_add(so_mul(E, 0x1.2fefa2p-17f), lf));   // ln2_hi, ln2_lo
}

// cos and sin of 2 pi k / 2^32: quadrant k >> 30 and the in-quadrant index are integers; the angle is
// folded to [0, pi/4] (index > 2^29 -> 2^30 - index, cos and sin swapped), where both are polynomials
BFLC_HD void dp_cossin(uint32_t k, float& c, float& s) {
  const uint32_t q = k >> 30;
  uint32_t r = k & 0x3FFFFFFFu;
  const bool fold = r > 0x20000000u;
  if (fold) r = 0x40000000u - r;
  const float x = so_mul(static_cast<float>(r), 0x1.921fb6p-30f);   // pi / 2^31
  const float x2 = so_mul(x, x);
  float ps = 0x1.71de3ap-19f;                          // 1/9!
  ps = so_add(so_mul(ps, x2), -0x1.a01a02p-13f);       // -1/7!
  ps = so_add(so_mul(ps, x2), 0x1.111112p-7f);         // 1/5!
  ps = so_add(so_mul(ps, x2), -0x1.555556p-3f);        // -1/3!
  const float sn = so_add(x, so_mul(so_mul(x, x2), ps));
  float pc = -0x1.27e4fcp-22f;                         // -1/10!
  pc = so_add(so_mul(pc, x2), 0x1.a01a02p-16f);        // 1/8!
  pc = so_add(so_mul(pc, x2), -0x1.6c16c2p-10f);       // -1/6!
  pc = so_add(so_mul(pc, x2), 0x1.555556p-5f);         // 1/4!
  pc = so_add(so_mul(pc, x2), -0.5f);
  const float cs = so_add(1.f, so_mul(x2, pc));
  const float cq = fold ? sn : cs, sq = fold ? cs : sn;
  c = q == 0 ? cq : q == 1 ? -sq : q == 2 ? -cq : sq;
  s = q == 0 ? sq : q == 1 ? cq : q == 2 ? -sq : -cq;
}

// Box-Muller on two 32-bit words: r = sqrt(-2 ln u), (r cos theta, r sin theta).  |z| <= sqrt(64 ln 2)
// ~ 6.66 (u >= 2^-32); the error against fp64 Box-Muller of the same words is stated in DESIGN.md.
BFLC_HD void dp_box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
  const float lu = dp_log_u(a);
  const float r = so_sqrt(so_sub(0.f, so_add(lu, lu)));
  float c, s;
  dp_cossin(b, c, s);
  z0 = so_mul(r, c);
  z1 = so_mul(r, s);
}

// The four standard normals of coordinates 4j .. 4j + 3 of round `epoch`: one Philox4x32-10 call,
// key = seed, counter = {j_lo, j_hi, epoch, site}, two Box-Muller pairs.  site: kDpSite (DP-FedAvg)
// or kDpsgdSite (DP-SGD, where `epoch` is the client's optimizer-step word).
BFLC_HD void dp_gauss4(uint64_t seed, uint32_t epoch, uint64_t j, float z[4], uint32_t site) {
  const philox::U4 w = philox::philox4x32_10(
      philox::U4{static_cast<uint32_t>(j), static_cast<uint32_t>(j >> 32), epoch, site},
      static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  dp_box_muller(w.x, w.y, z[0], z[1]);
  dp_box_muller(w.z, w.w, z[2], z[3]);
}

template <int MAXR>
BFLC_HD void run_consensus(const ConsensusIn<MAXR>& in, ConsensusOut<MAXR>& out) {
  const int n = in.n_ranks;
  // 0. median committee score per admitted trainer
  out.n_ranked = 0;
  for (int t = 0; t < n; ++t) {
    out.median[t] = 0.f;
    out.selected[t] = 0;
    out.weight[t] = 0.f;
    if (!in.admitted[t]) continue;
    float tmp[MAXR];
    int m = 0;
BFLC_UNROLL
    for (int c = 0; c < MAXR; ++c) {
      const bool ok = c < n && (in.role[c] & ROLE_COMM) && in.scored[c][t];
      tmp[c] = ok ? in.score[c][t] : __builtin_huge_valf();
      m += ok ? 1 : 0;
    }
    out.median[t] = median_of<MAXR>(tmp, m);
    out.order[out.n_ranked++] = t;
  }
  // 1. sort by (median desc, rank asc) -- insertion sort keeps it stable and tiny
  for (int i = 1; i < out.n_ranked; ++i) {
    const int x = out.order[i];
    int j = i - 1;
    while (j >= 0 && (out.median[out.order[j]] < out.median[x])) {
      out.order[j + 1] = out.order[j];
      --j;
    }
    out.order[j + 1] = x;
  }
  // 2-3. top-K, weights
  const int k = in.n_aggregate < out.n_ranked ? in.n_aggregate : out.n_ranked;
  out.n_selected = k;
  double wsum = 0.0;
  float cost = 0.f;
  for (int i = 0; i < k; ++i) {
    const int t = out.order[i];
    out.selected[t] = 1;
    double w = static_cast<double>(in.n_samples[t]);
    if (in.weight_by_score) w *= static_cast<double>(out.median[t]);
    out.weight[t] = static_cast<float>(w);
    wsum += w;
    cost += in.avg_cost[t];
  }
  if (k > 0 && wsum <= 0.0) {  // degenerate: all-zero scores -> fall back to uniform
    for (int i = 0; i < k; ++i) out.weight[out.order[i]] = 1.f;
    wsum = static_cast<double>(k);
  }
  for (int i = 0; i < k; ++i) {
    const int t = out.order[i];
    out.weight[t] = static_cast<float>(static_cast<double>(out.weight[t]) / wsum);
  }
  out.global_loss = k > 0 ? cost / static_cast<float>(k) : 0.f;
  // 5. re-election. Solo mode (a rank that is both trainer and committee) keeps its roles.
  bool solo = false;
  for (int r = 0; r < n; ++r)
    if ((in.role[r] & ROLE_TRAINER) && (in.role[r] & ROLE_COMM)) solo = true;
  for (int r = 0; r < n; ++r) out.role_after[r] = solo ? in.role[r] : ROLE_TRAINER;
  if (!solo) {
    int elected = 0;
    for (int i = 0; i < out.n_ranked && elected < in.n_comm; ++i) {
      out.role_after[out.order[i]] = ROLE_COMM;
      ++elected;
    }
    // not enough scored trainers to fill the committee: keep the lowest-ranked old members
    for (int r = 0; r < n && elected < in.n_comm; ++r) {
      if ((in.role[r] & ROLE_COMM) && out.role_after[r] != ROLE_COMM) {
        out.role_after[r] = ROLE_COMM;
        ++elected;
      }
    }
  }
}

}  // namespace bflc
