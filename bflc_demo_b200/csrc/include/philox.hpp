// Counter-based random numbers for dropout, one definition for the host and the device (the
// BFLC_HD style of consensus_math.hpp), so a g++ build and the kernels draw the same masks.
//
// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011): a
// 128-bit counter and a 64-bit key give 128 random bits, with no state between calls.
//
// Keep decisions.  A dropout mask is a pure function of (seed, step, site, coordinates); nothing is
// stored, so a backward pass regenerates exactly the forward's mask, and a CUDA graph replayed with
// a new step word draws new masks.  One Philox call decides 8 consecutive columns of one row:
//   key     = {seed low 32 bits, seed high 32 bits}
//   counter = {(row << 16) | (column >> 3), seq, (site << 8) | head, step}
// row and column are in-sequence coordinates (attention: query row i, key column j; hidden
// activations: token position i, feature column c), seq is the sequence's index in the batch and
// head is 0 for hidden activations.  No key depends on padding or packing.  Column t of the group
// (t = column & 7) takes the 16-bit uniform u = half (t & 1) of output word t >> 1, and is kept iff
// u >= thr, thr = round(p * 65536): the dropped fraction is thr / 65536, within 2^-17 of p.
// Limits: row, column >> 3 < 65536; head < 256; site < 2^24.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define BFLC_HD __host__ __device__ __forceinline__
#else
#define BFLC_HD inline
#endif

namespace bflc {
namespace philox {

struct U4 { uint32_t x, y, z, w; };

BFLC_HD uint32_t mulhi(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __umulhi(a, b);
#else
  return static_cast<uint32_t>((static_cast<uint64_t>(a) * b) >> 32);
#endif
}

BFLC_HD U4 philox4x32_10(U4 c, uint32_t k0, uint32_t k1) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = mulhi(M0, c.x), lo0 = M0 * c.x;
    const uint32_t hi1 = mulhi(M1, c.z), lo1 = M1 * c.z;
    c = U4{hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0};
    k0 += W0;
    k1 += W1;
  }
  return c;
}

// Everything a kernel needs to decide a keep; thr == 0 means no dropout.
struct Drop {
  uint32_t seed_lo, seed_hi;
  uint32_t step;     // the step word plus the caller's step add
  uint32_t site;
  uint32_t thr;      // round(p * 65536), at most 65535
  float scale;       // 1 / (1 - p), applied to kept values
};

BFLC_HD uint32_t threshold(float p) {
  const float t = p * 65536.f + 0.5f;
  const uint32_t u = t <= 0.f ? 0u : static_cast<uint32_t>(t);
  return u > 65535u ? 65535u : u;
}

// The 8 keep bits of columns 8 * group .. 8 * group + 7 of `row`: bit t = column 8 * group + t.
BFLC_HD uint32_t keep8(const Drop& d, uint32_t seq, uint32_t head, uint32_t row, uint32_t group) {
  const U4 r = philox4x32_10(U4{(row << 16) | group, seq, (d.site << 8) | head, d.step}, d.seed_lo, d.seed_hi);
  const uint32_t w[4] = {r.x, r.y, r.z, r.w};
  uint32_t bits = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int t = 0; t < 8; ++t) {
    const uint32_t u = (t & 1) ? (w[t >> 1] >> 16) : (w[t >> 1] & 0xFFFFu);
    bits |= static_cast<uint32_t>(u >= d.thr) << t;
  }
  return bits;
}

// One element: is (seq, head, row, col) kept?
BFLC_HD bool keep(const Drop& d, uint32_t seq, uint32_t head, uint32_t row, uint32_t col) {
  return (keep8(d, seq, head, row, col >> 3) >> (col & 7)) & 1u;
}

}  // namespace philox
}  // namespace bflc
