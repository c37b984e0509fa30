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
//     server_step), default off = the aggregate is the new global model.
#pragma once
#include <cmath>
#include <cstdint>

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
// block record's word also carries the server optimizer (ServerOpt below) in bits 16..23; "none"
// leaves every word unchanged.
BFLC_HD uint32_t agg_word(int rule, int trim, int server_opt = 0) {
  return static_cast<uint32_t>(rule) | (rule == AGG_TRIMMED_MEAN ? static_cast<uint32_t>(trim) << 8 : 0u) |
         static_cast<uint32_t>(server_opt) << 16;
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
