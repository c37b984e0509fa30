// DP-SGD (Abadi et al. 2016) with book-keeping clipping (ops/dpsgd.py): per-example gradient norms,
// certified clip factors, per-example row scaling, deterministic bias column sums and the client's
// Gaussian noise.
//
// A weight gradient over B examples of R rows each is G = sum_n A_n^T Bm_n, A_n / Bm_n the n-th R-row
// blocks of A [B*R, a] and Bm [B*R, b].  The per-example part ||A_n^T Bm_n||_F^2 never materialises:
// k_pe_norm keeps one 64 x 64 product tile of it in wgmma accumulators (64 columns of A as the M
// dimension, 64 columns of Bm as N -- a convolution's patches, with a column of ones for its bias --, the
// example's rows as K, both operands MN-major, read straight from the row-major activations) and its
// epilogue squares and reduces the tile to one fp32 partial per (tile, example).  R = 1 sites (whole-row
// layers) use the identity ||dz x^T||^2 + ||dz||^2 = ||dz||^2 (||x||^2 + 1) in k_pe_rows instead.  Every sum runs in a fixed
// order, so the factors are bit-reproducible; k_dpsgd_clip is written with the correctly rounded so_*
// operations so that ops/dpsgd.py's numpy mirror computes the same bits.
#include <cuda_bf16.h>

#include "bflc_kernels.h"
#include "consensus_math.hpp"
#include "sm100_ptx.cuh"
#include "wgmma.cuh"

namespace bflc {

namespace {

typedef __nv_bfloat16 bf16;
constexpr int kNT = 128;   // k_pe_norm: one warpgroup

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// 8 consecutive bf16 of row `row`, columns [c0, c0 + 8) of X; zero outside the matrix (ok = row inside)
__device__ __forceinline__ uint4 load8(const bf16* __restrict__ X, long long ld, long long row, bool ok, int c0,
                                       int cols, bool vec) {
  if (!ok || c0 >= cols) return make_uint4(0u, 0u, 0u, 0u);
  const bf16* p = X + row * ld + c0;
  if (vec && c0 + 8 <= cols) return __ldg(reinterpret_cast<const uint4*>(p));
  uint32_t h[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) h[e] = c0 + e < cols ? static_cast<uint32_t>(__bfloat16_as_ushort(p[e])) : 0u;
  return make_uint4(h[0] | (h[1] << 16), h[2] | (h[3] << 16), h[4] | (h[5] << 16), h[6] | (h[7] << 16));
}

// 8 bf16 of columns [c0, c0 + 8) with a 1 at column `one` (a site bias' extra operand column; -1: none)
__device__ __forceinline__ uint4 with_one(uint4 r, int c0, int one) {
  const int e = one - c0;
  if (one < 0 || e < 0 || e >= 8) return r;
  const uint32_t v = 0x3F80u << ((e & 1) * 16);   // bf16 1.0
  r.x |= (e >> 1) == 0 ? v : 0u;
  r.y |= (e >> 1) == 1 ? v : 0u;
  r.z |= (e >> 1) == 2 ? v : 0u;
  r.w |= (e >> 1) == 3 ? v : 0u;
  return r;
}

// the 64-token chunk starting at token t0 of example rows [row0, row0 + R): 512 16-byte pieces per
// operand, four per thread; piece (t, c) is token t, columns 8c .. 8c + 7 of the tile (A from col0, Bm
// from colb; Bm's column `one` reads 1 on the example's rows)
__device__ __forceinline__ void fetch(uint4 (&ra)[4], uint4 (&rb)[4], const bf16* __restrict__ A, long long lda,
                                      int a_cols, const bf16* __restrict__ Bm, long long ldb, int b_cols,
                                      long long row0, int R, int t0, int col0, int colb, int one, bool vec_a,
                                      bool vec_b) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = threadIdx.x + kNT * i, t = idx >> 3, c = idx & 7;
    const bool ok = t0 + t < R;
    ra[i] = load8(A, lda, row0 + t0 + t, ok, col0 + 8 * c, a_cols, vec_a);
    rb[i] = load8(Bm, ldb, row0 + t0 + t, ok, colb + 8 * c, b_cols, vec_b);
    if (ok) rb[i] = with_one(rb[i], colb + 8 * c, one);
  }
}

// Packed batches (SEG): example n owns rows [cu[n], cu[n + 1]) instead of [n R, (n + 1) R).  seg_rows checks
// what the host cannot check without a sync: cu[0] == 0, 0 <= L_n <= max_rows and cu[n + 1] <= rows.  An example
// that fails it gets a NaN partial, so k_dpsgd_clip drops it and counts it.
__device__ __forceinline__ bool seg_rows(const int32_t* __restrict__ cu, int n, long long rows, int max_rows,
                                         long long& row0, int& L) {
  row0 = cu[n];
  const long long end = cu[n + 1];
  L = static_cast<int>(end - row0);
  return cu[0] == 0 && L >= 0 && L <= max_rows && end <= rows;
}

// grid (a_tiles * b_tiles, B): out[tile * B + n] = sum over the tile's 64 x 64 entries of (A_n^T [Bm_n | 1])^2,
// tile = ta + a_tiles * tb covering columns [64 ta, 64 ta + 64) of A and [64 tb, 64 tb + 64) of Bm, whose
// column `one` (= b_cols, a site bias; -1: none) reads 1.  No limit on R: rows past it are zero-filled.
// SEG: the K loop runs over example n's own L_n rows (cu, rows: seg_rows).
template <bool SEG>
__device__ __forceinline__ void pe_norm_body(const bf16* __restrict__ A, long long lda, int a_cols,
                                             const bf16* __restrict__ Bm, long long ldb, int b_cols, int R, int n_ex,
                                             float* __restrict__ out, int vec_a, int vec_b, int a_tiles, int one,
                                             const int32_t* __restrict__ cu, long long rows) {
  // MN-major 128B-swizzled operand tiles [64 tokens][64 columns]: token t is the 128-byte row t, its
  // 16-byte piece c sits at piece c ^ (t & 7)
  __shared__ __align__(1024) uint8_t sm[2 * 8192];
  __shared__ float red[4];
  const int n = blockIdx.y, col0 = (blockIdx.x % a_tiles) * 64, colb = (blockIdx.x / a_tiles) * 64;
  long long row0;
  if constexpr (SEG) {
    if (!seg_rows(cu, n, rows, INT_MAX, row0, R)) {
      if (threadIdx.x == 0) out[static_cast<long long>(blockIdx.x) * n_ex + n] = __int_as_float(0x7FC00000);
      return;
    }
  } else {
    row0 = static_cast<long long>(n) * R;
  }
  const uint32_t sa = ptx::smem_u32(sm), sb = sa + 8192u;
  float d[32];
  wg::zero(d);
  uint4 ra[4], rb[4];
  fetch(ra, rb, A, lda, a_cols, Bm, ldb, b_cols, row0, R, 0, col0, colb, one, vec_a != 0, vec_b != 0);
  for (int t0 = 0; t0 < R; t0 += 64) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = threadIdx.x + kNT * i, t = idx >> 3, c = idx & 7;
      const int off = t * 128 + ((c ^ (t & 7)) << 4);
      *reinterpret_cast<uint4*>(sm + off) = ra[i];
      *reinterpret_cast<uint4*>(sm + 8192 + off) = rb[i];
    }
    ptx::fence_proxy_async_smem();
    __syncthreads();
    wg::fence();
#pragma unroll
    for (uint32_t ks = 0; ks < 4; ++ks)
      wg::mma_bf16<64, 1, 1>(d, wg::desc(sa + ks * 2048u, 8192), wg::desc(sb + ks * 2048u, 8192),
                             (t0 > 0 || ks > 0) ? 1u : 0u);
    wg::commit();
    if (t0 + 64 < R)   // the next chunk's loads overlap the MMAs
      fetch(ra, rb, A, lda, a_cols, Bm, ldb, b_cols, row0, R, t0 + 64, col0, colb, one, vec_a != 0, vec_b != 0);
    wg::wait<0>();
    wg::reg_fence(d);
    __syncthreads();   // every warp's MMAs are done before the tiles are overwritten
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) s = fmaf(d[i], d[i], s);
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) out[static_cast<long long>(blockIdx.x) * n_ex + n] = ((red[0] + red[1]) + red[2]) + red[3];
}

__global__ void __launch_bounds__(kNT) k_pe_norm(const bf16* __restrict__ A, long long lda, int a_cols,
                                                 const bf16* __restrict__ Bm, long long ldb, int b_cols, int R,
                                                 int n_ex, float* __restrict__ out, int vec_a, int vec_b,
                                                 int a_tiles, int one) {
  pe_norm_body<false>(A, lda, a_cols, Bm, ldb, b_cols, R, n_ex, out, vec_a, vec_b, a_tiles, one, nullptr, 0);
}

__global__ void __launch_bounds__(kNT) k_packed_norm(const bf16* __restrict__ A, long long lda, int a_cols,
                                                     const bf16* __restrict__ Bm, long long ldb, int b_cols,
                                                     int n_ex, float* __restrict__ out, int vec_a, int vec_b,
                                                     int a_tiles, int one, const int32_t* __restrict__ cu,
                                                     long long rows) {
  pe_norm_body<true>(A, lda, a_cols, Bm, ldb, b_cols, 0, n_ex, out, vec_a, vec_b, a_tiles, one, cu, rows);
}

// ---------------------------------------------------------------- Gram ("ghost") norms
// ||P_n^T Q_n||_F^2 = sum_{t,t'} (p_t . p_t') (q_t . q_t') for sites whose two sides are both wider than
// 64.  One CTA owns the 64 x 64 row-tile pair (i, j) of example n: Gp = P_i P_j^T and Gq = Q_i Q_j^T are
// two m64n64k16 accumulators with K-major operands (the row-major activations as they are), sharing one
// fragment layout, so (Gp, Gq) products are lane-local.  P is dense, one-hot ([id_t == id_t'], from
// int32 ids) or a gather (P_t[id_t'], the tied head's cross term); Q is dense, extended by a 1 when the
// site has a bias (Gq + 1).  Rows past R are zero-filled.
struct GramArgs {
  const bf16* p1;
  const bf16* p2;
  long long ldp1, ldp2;
  int kp;
  const int32_t* id1;
  const int32_t* id2;
  const bf16* q1;
  const bf16* q2;
  long long ldq1, ldq2;
  int kq;
  int R, n_ex, tiles, mode, sym;
  float bias;
  float* out;
  int vec_p, vec_q;
};
constexpr int kGramDense = 0, kGramOneHot = 1, kGramGather = 2;

// d = X1[r1 .. r1 + n1) X2[r2 .. r2 + n2)^T over K columns, in 64-column chunks; rows past n zero-filled
__device__ __forceinline__ void gram_acc(float (&d)[32], uint8_t* sm, uint32_t sa, const bf16* __restrict__ X1,
                                         long long ld1, const bf16* __restrict__ X2, long long ld2, int K,
                                         long long r1, int n1, long long r2, int n2, bool same, bool vec) {
  const uint32_t sb = same ? sa : sa + 8192u;
  uint4 ra[4], rb[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = threadIdx.x + kNT * i, t = idx >> 3, c = idx & 7;
    ra[i] = load8(X1, ld1, r1 + t, t < n1, 8 * c, K, vec);
    rb[i] = same ? ra[i] : load8(X2, ld2, r2 + t, t < n2, 8 * c, K, vec);
  }
  for (int k0 = 0; k0 < K; k0 += 64) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = threadIdx.x + kNT * i, t = idx >> 3, c = idx & 7;
      const int off = t * 128 + ((c ^ (t & 7)) << 4);
      *reinterpret_cast<uint4*>(sm + off) = ra[i];
      if (!same) *reinterpret_cast<uint4*>(sm + 8192 + off) = rb[i];
    }
    ptx::fence_proxy_async_smem();
    __syncthreads();
    wg::fence();
#pragma unroll
    for (uint32_t ks = 0; ks < 4; ++ks)
      wg::mma_bf16<64, 0, 0>(d, wg::desc(sa + ks * 32u, 16), wg::desc(sb + ks * 32u, 16), (k0 > 0 || ks > 0) ? 1u : 0u);
    wg::commit();
    if (k0 + 64 < K) {   // the next chunk's loads overlap the MMAs
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int idx = threadIdx.x + kNT * i, t = idx >> 3, c = idx & 7;
        ra[i] = load8(X1, ld1, r1 + t, t < n1, k0 + 64 + 8 * c, K, vec);
        rb[i] = same ? ra[i] : load8(X2, ld2, r2 + t, t < n2, k0 + 64 + 8 * c, K, vec);
      }
    }
    wg::wait<0>();
    wg::reg_fence(d);
    __syncthreads();   // every warp's MMAs are done before the tiles are overwritten
  }
}

// grid (pairs, B): out[pair * B + n] = w sum over the pair's 64 x 64 entries of Gp Gq, w = 2 off the
// diagonal (sym: pairs i <= j of one row set; else every (i, j) of two row sets, the cross term)
// SEG: the pairs are those of g.tiles = ceil(max_len / 64) tiles; example n's tiles start at its first row,
// and a CTA whose pair lies past its ceil(L_n / 64) tiles stores +0 before any operand load.  Its nonzero
// partials keep their order, so every sum over them equals the example's own uniform launch at R = L_n.
template <bool SEG>
__device__ __forceinline__ void pe_gram_body(const GramArgs& g, const int32_t* __restrict__ cu, long long rows) {
  __shared__ __align__(1024) uint8_t sm[2 * 8192];
  __shared__ float red[4];
  const int n = blockIdx.y;
  int ti = 0, tj = blockIdx.x;
  if (g.sym) {
    while (tj >= g.tiles - ti) tj -= g.tiles - ti++;
    tj += ti;
  } else {
    ti = tj / g.tiles;
    tj -= ti * g.tiles;
  }
  long long row0;
  int R;
  if constexpr (SEG) {
    float* o = g.out + static_cast<long long>(blockIdx.x) * g.n_ex + n;
    if (!seg_rows(cu, n, rows, 64 * g.tiles, row0, R)) {
      if (threadIdx.x == 0) *o = __int_as_float(0x7FC00000);
      return;
    }
    if (64 * ti >= R || 64 * tj >= R) {
      if (threadIdx.x == 0) *o = 0.f;
      return;
    }
  } else {
    row0 = static_cast<long long>(n) * g.R;
    R = g.R;
  }
  const int ni = min(64, R - 64 * ti), nj = min(64, R - 64 * tj);
  const bool same = g.sym && ti == tj;
  const uint32_t sa = ptx::smem_u32(sm);
  float dp[32], dq[32];
  if (g.mode == kGramDense)
    gram_acc(dp, sm, sa, g.p1, g.ldp1, g.p2, g.ldp2, g.kp, row0 + 64 * ti, ni, row0 + 64 * tj, nj, same,
             g.vec_p != 0);
  gram_acc(dq, sm, sa, g.q1, g.ldq1, g.q2, g.ldq2, g.kq, row0 + 64 * ti, ni, row0 + 64 * tj, nj, same,
           g.vec_q != 0);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int r = 16 * w + (l >> 2) + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
    float gp;
    if (g.mode == kGramDense) {
      gp = dp[i];
    } else if (r < ni && c < nj) {
      const long long t = row0 + 64 * ti + r, u = row0 + 64 * tj + c;
      gp = g.mode == kGramOneHot ? (g.id1[t] == g.id2[u] ? 1.f : 0.f)
                                 : __bfloat162float(g.p1[t * g.ldp1 + g.id2[u]]);
    } else {
      gp = 0.f;
    }
    s = fmaf(gp, so_add(dq[i], g.bias), s);
  }
  s = warp_sum(s);
  if (l == 0) red[w] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    const float t = ((red[0] + red[1]) + red[2]) + red[3];
    g.out[static_cast<long long>(blockIdx.x) * g.n_ex + n] = same ? t : 2.f * t;
  }
}

__global__ void __launch_bounds__(kNT) k_pe_gram(const GramArgs g) { pe_gram_body<false>(g, nullptr, 0); }

__global__ void __launch_bounds__(kNT) k_packed_gram(const GramArgs g, const int32_t* __restrict__ cu,
                                                     long long rows) {
  pe_gram_body<true>(g, cu, rows);
}

// ---------------------------------------------------------------- layer norms
// xhat exactly as the release computes it (no contraction): (x - mean) * rstd
__device__ __forceinline__ float ln_xhat(const bf16* __restrict__ x, long long i, float m, float rs) {
  return __fmul_rn(__fsub_rn(__bfloat162float(x[i]), m), rs);
}

// one block per example n over its R rows of dy, x [rows, C] (mean, rstd per row):
// sq[n] = ||sum_t dy_t . xhat_t||^2 + ||sum_t dy_t||^2 (gamma and beta), each column's sums in row order;
// ab[n] = sum_t ||dy_t|| (max_c |xhat_tc| + 1) in row order
constexpr int kMaxRowsR = 512;
constexpr int kMaxRowsAbs = 1024;   // k_pe_rows: a convolution's output positions per example (32 x 32)
// SEG: over example n's own rows [cu[n], cu[n + 1]) (seg_rows)
template <bool SEG>
__device__ __forceinline__ void pe_ln_body(const bf16* __restrict__ dy, const bf16* __restrict__ x, int C, int R,
                                           const float* __restrict__ mean, const float* __restrict__ rstd,
                                           float* __restrict__ sq_out, float* __restrict__ ab_out,
                                           const int32_t* __restrict__ cu, long long rows) {
  __shared__ float term[kMaxRowsR];
  __shared__ float red[8];
  const int n = blockIdx.x, w = threadIdx.x >> 5, l = threadIdx.x & 31;
  long long row0;
  if constexpr (SEG) {
    if (!seg_rows(cu, n, rows, kMaxRowsR, row0, R)) {
      if (threadIdx.x == 0) sq_out[n] = ab_out[n] = __int_as_float(0x7FC00000);
      return;
    }
  } else {
    row0 = static_cast<long long>(n) * R;
  }
  for (int t = w; t < R; t += 8) {
    const long long r = row0 + t;
    const float m = mean[r], rs = rstd[r];
    float dd = 0.f, mx = 0.f;
    for (int c = l; c < C; c += 32) {
      const float v = __bfloat162float(dy[r * C + c]);
      dd = fmaf(v, v, dd);
      mx = fmaxf(mx, fabsf(ln_xhat(x, r * C + c, m, rs)));
    }
    dd = warp_sum(dd);
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (l == 0) term[t] = so_mul(so_sqrt(dd), so_add(mx, 1.f));
  }
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += 256) {
    float gg = 0.f, gb = 0.f;
    for (int t = 0; t < R; ++t) {
      const long long r = row0 + t;
      const float v = __bfloat162float(dy[r * C + c]);
      gg = fmaf(v, ln_xhat(x, r * C + c, mean[r], rstd[r]), gg);
      gb = so_add(gb, v);
    }
    s = fmaf(gg, gg, fmaf(gb, gb, s));
  }
  s = warp_sum(s);
  if (l == 0) red[w] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float q = 0.f, a = 0.f;
    for (int k = 0; k < 8; ++k) q = so_add(q, red[k]);
    for (int t = 0; t < R; ++t) a = so_add(a, term[t]);
    sq_out[n] = q;
    ab_out[n] = a;
  }
}

__global__ void __launch_bounds__(256) k_pe_ln(const bf16* __restrict__ dy, const bf16* __restrict__ x, int C, int R,
                                               const float* __restrict__ mean, const float* __restrict__ rstd,
                                               float* __restrict__ sq_out, float* __restrict__ ab_out) {
  pe_ln_body<false>(dy, x, C, R, mean, rstd, sq_out, ab_out, nullptr, 0);
}

__global__ void __launch_bounds__(256) k_packed_ln(const bf16* __restrict__ dy, const bf16* __restrict__ x, int C,
                                                   const float* __restrict__ mean, const float* __restrict__ rstd,
                                                   float* __restrict__ sq_out, float* __restrict__ ab_out,
                                                   const int32_t* __restrict__ cu, long long rows) {
  pe_ln_body<true>(dy, x, C, 0, mean, rstd, sq_out, ab_out, cu, rows);
}

// gg[j] += sum_r S[r, j] xhat[r, j], gb[j] += sum_r S[r, j] for the clipped rows S = bf16(c dy): 32 columns x
// 16 row lanes per block as k_colsum_fixed; a dropped example's rows (c = 0) are skipped, their xhat may not
// be finite.  SEG: row r's example is seg[r] (row_factor)
template <bool SEG>
__device__ __forceinline__ float row_factor(const float* __restrict__ c, long long r, int R,
                                            const int32_t* __restrict__ seg, int n_ex) {
  if constexpr (SEG) {
    const int e = seg[r];
    return static_cast<unsigned>(e) < static_cast<unsigned>(n_ex) ? c[e] : 0.f;   // out of range: dropped
  } else {
    return c[r / R];
  }
}

template <bool SEG>
__device__ __forceinline__ void ln_release_body(const bf16* __restrict__ S, long long lds, const bf16* __restrict__ x,
                                                const float* __restrict__ mean, const float* __restrict__ rstd,
                                                long long rows, int C, const float* __restrict__ cf, int R,
                                                float* __restrict__ gg, float* __restrict__ gb,
                                                const int32_t* __restrict__ seg, int n_ex) {
  __shared__ float sg[16][33], sb[16][33];
  const int lane = threadIdx.x & 31, rl = threadIdx.x >> 5, j = blockIdx.x * 32 + lane;
  float a = 0.f, b = 0.f;
  if (j < C)
    for (long long r = rl; r < rows; r += 16) {
      if ((dp_bits(row_factor<SEG>(cf, r, R, seg, n_ex)) & 0x7FFFFFFFu) == 0u) continue;
      const float v = __bfloat162float(S[r * lds + j]);
      a = so_add(a, so_mul(v, ln_xhat(x, r * C + j, mean[r], rstd[r])));
      b = so_add(b, v);
    }
  sg[rl][lane] = a;
  sb[rl][lane] = b;
  __syncthreads();
  if (rl == 0 && j < C) {
    float ta = sg[0][lane], tb = sb[0][lane];
#pragma unroll
    for (int k = 1; k < 16; ++k) {
      ta = so_add(ta, sg[k][lane]);
      tb = so_add(tb, sb[k][lane]);
    }
    gg[j] = so_add(gg[j], ta);
    gb[j] = so_add(gb[j], tb);
  }
}

__global__ void __launch_bounds__(512) k_ln_release(const bf16* __restrict__ S, long long lds,
                                                    const bf16* __restrict__ x, const float* __restrict__ mean,
                                                    const float* __restrict__ rstd, long long rows, int C,
                                                    const float* __restrict__ cf, int R, float* __restrict__ gg,
                                                    float* __restrict__ gb) {
  ln_release_body<false>(S, lds, x, mean, rstd, rows, C, cf, R, gg, gb, nullptr, 0);
}

__global__ void __launch_bounds__(512) k_packed_ln_release(const bf16* __restrict__ S, long long lds,
                                                           const bf16* __restrict__ x, const float* __restrict__ mean,
                                                           const float* __restrict__ rstd, long long rows, int C,
                                                           const float* __restrict__ cf, float* __restrict__ gg,
                                                           float* __restrict__ gb, const int32_t* __restrict__ seg,
                                                           int n_ex) {
  ln_release_body<true>(S, lds, x, mean, rstd, rows, C, cf, 1, gg, gb, seg, n_ex);
}

// ---------------------------------------------------------------- embeddings
// perm[rank_r] = r, rank_r = #{r' : id_r' < id_r} + #{r' < r : id_r' == id_r}: a stable sort of the ids
__global__ void k_id_rank(const int32_t* __restrict__ ids, int rows, int32_t* __restrict__ perm) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int v = ids[r];
  int k = 0;
  for (int q = 0; q < rows; ++q) {
    const int u = ids[q];
    k += (u < v || (u == v && q < r)) ? 1 : 0;
  }
  perm[k] = r;
}

// one block per sorted position p; the first position of each id v sums its rows of S in row order into
// table row v: G[v, j] += sum S[r, j].  One writer per element, no atomics.
__global__ void __launch_bounds__(128) k_seg_release(const bf16* __restrict__ S, long long lds, int C,
                                                     const int32_t* __restrict__ ids,
                                                     const int32_t* __restrict__ perm, int rows,
                                                     float* __restrict__ G, long long ldg) {
  const int p = blockIdx.x;
  const int v = ids[perm[p]];
  if (p > 0 && ids[perm[p - 1]] == v) return;
  int end = p + 1;
  while (end < rows && ids[perm[end]] == v) ++end;
  for (int j = threadIdx.x; j < C; j += 128) {
    float s = 0.f;
    for (int q = p; q < end; ++q) s = so_add(s, __bfloat162float(S[static_cast<long long>(perm[q]) * lds + j]));
    float* o = G + static_cast<long long>(v) * ldg + j;
    *o = so_add(*o, s);
  }
}

// one block of min(R, 8) warps per example n (R <= kMaxRowsAbs).  Row t of the example gets ra_t = ||A_t||^2 and
// rb_t = ||Bm_t||^2 + bias; abs_out[n] = sum_t sqrt(ra_t) sqrt(rb_t) in token order, and for R = 1
// sq_out[n] = ra_0 rb_0 (the squared norm of the row's weight-and-bias gradient).  One warp forms each row's
// term and one thread sums them in order, so the bits do not depend on the warp count.
// SEG: over example n's own rows [cu[n], cu[n + 1]) (seg_rows), no sq_out
template <bool SEG>
__device__ __forceinline__ void pe_rows_body(const bf16* __restrict__ A, long long lda, int a_cols,
                                             const bf16* __restrict__ Bm, long long ldb, int b_cols, int R,
                                             float bias, float* __restrict__ sq_out, float* __restrict__ abs_out,
                                             const int32_t* __restrict__ cu, long long rows) {
  __shared__ float term[kMaxRowsAbs];
  const int n = blockIdx.x, w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  long long row0 = 0;
  if constexpr (SEG) {
    if (!seg_rows(cu, n, rows, kMaxRowsAbs, row0, R)) {
      if (threadIdx.x == 0) abs_out[n] = __int_as_float(0x7FC00000);
      return;
    }
  }
  for (int t = w; t < R; t += nw) {
    const long long row = SEG ? row0 + t : static_cast<long long>(n) * R + t;
    float a = 0.f, b = 0.f;
    for (int c = l; c < a_cols; c += 32) {
      const float v = __bfloat162float(A[row * lda + c]);
      a = fmaf(v, v, a);
    }
    for (int c = l; c < b_cols; c += 32) {
      const float v = __bfloat162float(Bm[row * ldb + c]);
      b = fmaf(v, v, b);
    }
    a = warp_sum(a);
    b = so_add(warp_sum(b), bias);
    if (l == 0) {
      term[t] = so_mul(so_sqrt(a), so_sqrt(b));
      if constexpr (!SEG)
        if (R == 1 && sq_out != nullptr) sq_out[n] = so_mul(a, b);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int t = 0; t < R; ++t) s = so_add(s, term[t]);
    abs_out[n] = s;
  }
}

__global__ void __launch_bounds__(256) k_pe_rows(const bf16* __restrict__ A, long long lda, int a_cols,
                                                 const bf16* __restrict__ Bm, long long ldb, int b_cols, int R,
                                                 float bias, float* __restrict__ sq_out, float* __restrict__ abs_out) {
  pe_rows_body<false>(A, lda, a_cols, Bm, ldb, b_cols, R, bias, sq_out, abs_out, nullptr, 0);
}

__global__ void __launch_bounds__(256) k_packed_rows(const bf16* __restrict__ A, long long lda, int a_cols,
                                                     const bf16* __restrict__ Bm, long long ldb, int b_cols,
                                                     float bias, float* __restrict__ abs_out,
                                                     const int32_t* __restrict__ cu, long long rows) {
  pe_rows_body<true>(A, lda, a_cols, Bm, ldb, b_cols, 0, bias, nullptr, abs_out, cu, rows);
}

// the same abs term for an implicit-GEMM convolution site, whose patches p_t are never formed: one block of
// min(R, 8) warps per example; ||p_t||^2 = sum over the taps (r, s) inside the image, in tap order, of
// ||x_pix||^2 (a padding tap contributes 0), the stride applied; abs_out[n] = sum_t ||dz_t|| sqrt(||p_t||^2 +
// bias) in row order
__global__ void __launch_bounds__(256, 1) k_patch_rows(const bf16* __restrict__ dz, long long ldz, int Cout,
                                                    const bf16* __restrict__ x, int H, int W, int C, int OH, int OW,
                                                    int KH, int KW, int stride, int pad, float bias,
                                                    float* __restrict__ abs_out) {
  __shared__ float term[kMaxRowsAbs];
  const int n = blockIdx.x, w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5, R = OH * OW;
  for (int t = w; t < R; t += nw) {
    const long long row = static_cast<long long>(n) * R + t;
    const int oh = t / OW, ow = t - oh * OW;
    float a = 0.f, b = 0.f;
    for (int c = l; c < Cout; c += 32) {
      const float v = __bfloat162float(dz[row * ldz + c]);
      a = fmaf(v, v, a);
    }
    for (int r = 0; r < KH; ++r) {
      const int h = oh * stride + r - pad;
      for (int q = 0; q < KW; ++q) {
        const int v0 = ow * stride + q - pad;
        if (h < 0 || h >= H || v0 < 0 || v0 >= W) continue;   // warp-uniform
        const bf16* px = x + ((static_cast<long long>(n) * H + h) * W + v0) * C;
        float e = 0.f;
        for (int c = l; c < C; c += 32) {
          const float v = __bfloat162float(px[c]);
          e = fmaf(v, v, e);
        }
        b = so_add(b, warp_sum(e));
      }
    }
    a = warp_sum(a);
    if (l == 0) term[t] = so_mul(so_sqrt(a), so_sqrt(so_add(b, bias)));
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int t = 0; t < R; ++t) s = so_add(s, term[t]);
    abs_out[n] = s;
  }
}

// c[n] from the sites' partials sq [n_sq][B] and abs [n_ab][B] (DESIGN.md, "DP-SGD"):
//   norm = sqrt(sum sq), bound = (B norm) (1 + gamma) + (B abs) (u + gamma),
//   c = 0 for a non-finite bound (the example is dropped and counted), else 1 if bound <= C, else C / bound
// (dpsgd_clip_factor, consensus_math.hpp, which the persistent trainer's DP-SGD entry shares)
// With Gram sites (kap != nullptr, kap[i] > 0 for the abs rows of a Gram site), their cancellation slack
// kap_i abs_i^2 is folded in under the root: norm = sqrt(sum sq + sum_i kap_i abs_i^2).
// n_valid (nullable): examples n >= *n_valid are padding slots of a Poisson batch: c = 0, not counted as dropped.
__global__ void k_dpsgd_clip(const float* __restrict__ sq, int n_sq, const float* __restrict__ ab, int n_ab,
                             const float* __restrict__ kap, int n_ex, float bsz, float clip, float* __restrict__ c,
                             int* __restrict__ dropped, const int* __restrict__ n_valid) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_ex) return;
  if (n_valid != nullptr && n >= *n_valid) {
    c[n] = 0.f;
    return;
  }
  float s = 0.f, a = 0.f;
  for (int i = 0; i < n_sq; ++i) s = so_add(s, sq[static_cast<long long>(i) * n_ex + n]);
  for (int i = 0; i < n_ab; ++i) a = so_add(a, ab[static_cast<long long>(i) * n_ex + n]);
  if (kap != nullptr) {
    float k = 0.f;
    for (int i = 0; i < n_ab; ++i) {
      if (kap[i] == 0.f) continue;
      const float v = ab[static_cast<long long>(i) * n_ex + n];
      k = so_add(k, so_mul(kap[i], so_mul(v, v)));
    }
    s = so_add(s, k);
  }
  bool drop;
  c[n] = dpsgd_clip_factor(s, a, bsz, clip, &drop);
  if (drop) atomicAdd(dropped, 1);
}

// out[r, j] = bf16(X[r, j] * c[r / R]) (mask_only: X[r, j] unscaled), and exactly +0 where c[r / R] is 0:
// a dropped example's rows may hold NaN or inf, which a product with 0 would keep.  SEG: c[seg[r]]
template <bool SEG>
__device__ __forceinline__ void scale_rows_body(const bf16* __restrict__ X, long long ldx, bf16* __restrict__ out,
                                                long long ldo, long long rows, int cols, const float* __restrict__ c,
                                                int R, int mask_only, const int32_t* __restrict__ seg, int n_ex) {
  const long long total = rows * cols;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / cols;
    const int j = static_cast<int>(i - r * cols);
    const float cr = row_factor<SEG>(c, r, R, seg, n_ex);
    const bf16 x = X[r * ldx + j];
    out[r * ldo + j] = (dp_bits(cr) & 0x7FFFFFFFu) == 0u ? __float2bfloat16_rn(0.f)
                       : mask_only                        ? x
                                                          : __float2bfloat16_rn(so_mul(__bfloat162float(x), cr));
  }
}

__global__ void k_scale_rows(const bf16* __restrict__ X, long long ldx, bf16* __restrict__ out, long long ldo,
                             long long rows, int cols, const float* __restrict__ c, int R, int mask_only) {
  scale_rows_body<false>(X, ldx, out, ldo, rows, cols, c, R, mask_only, nullptr, 0);
}

__global__ void k_packed_scale_rows(const bf16* __restrict__ X, long long ldx, bf16* __restrict__ out, long long ldo,
                                    long long rows, int cols, const float* __restrict__ c, int mask_only,
                                    const int32_t* __restrict__ seg, int n_ex) {
  scale_rows_body<true>(X, ldx, out, ldo, rows, cols, c, 1, mask_only, seg, n_ex);
}

// g[j] += sum_r X[r, j]: 32 columns x 16 row lanes per block, each lane's rows in order, then the 16
// lane sums in order -- the same bits on every run (the atomics of act_bwd_colsum are not)
__global__ void __launch_bounds__(512) k_colsum_fixed(const bf16* __restrict__ X, long long ld, long long rows,
                                                      int cols, float* __restrict__ g) {
  __shared__ float sh[16][33];
  const int lane = threadIdx.x & 31, rl = threadIdx.x >> 5, j = blockIdx.x * 32 + lane;
  float s = 0.f;
  if (j < cols)
    for (long long r = rl; r < rows; r += 16) s = so_add(s, __bfloat162float(X[r * ld + j]));
  sh[rl][lane] = s;
  __syncthreads();
  if (rl == 0 && j < cols) {
    float t = sh[0][lane];
#pragma unroll
    for (int k = 1; k < 16; ++k) t = so_add(t, sh[k][lane]);
    g[j] = so_add(g[j], t);
  }
}

// g[i] += sigma * xi_i, xi_i = dp_gauss4(seed, *step + add, i / 4, kDpsgdSite)[i % 4]
__global__ void k_dpsgd_noise(float* __restrict__ g, long long P, uint64_t seed, const int32_t* __restrict__ step,
                              uint32_t add, float sigma) {
  const uint32_t word = static_cast<uint32_t>(*step) + add;
  const long long n4 = (P + 3) / 4;
  for (long long j = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; j < n4;
       j += static_cast<long long>(gridDim.x) * blockDim.x) {
    float z[4];
    dp_gauss4(seed, word, static_cast<uint64_t>(j), z, kDpsgdSite);
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (4 * j + q < P) g[4 * j + q] = so_add(g[4 * j + q], so_mul(sigma, z[q]));
  }
}

// ---------------------------------------------------------------- Poisson sampling
// One CTA per local step i: word = *step + i; record j in [0, S) is sampled iff u_j < thr, u_j word j % 4 of
// philox4x32_10({j / 4, 0, word, kDpsgdSampleSite}, seed).  Each pass covers 4 * kSampleNT records (one Philox
// call per thread); a block-wide exclusive scan of the per-thread counts places the sampled records in record
// order, no atomics.  The first `cap` are kept; slots past the count point at record 0 (padding).
constexpr int kSampleNT = 256;
__global__ void __launch_bounds__(kSampleNT) k_dpsgd_poisson_sample(uint64_t seed, const int32_t* __restrict__ step,
                                                                    int S, uint32_t thr, int cap,
                                                                    int32_t* __restrict__ idx,
                                                                    int32_t* __restrict__ count,
                                                                    int32_t* __restrict__ overflow) {
  __shared__ int warp_tot[kSampleNT / 32];
  const uint32_t word = static_cast<uint32_t>(*step) + blockIdx.x;
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  int32_t* out = idx + static_cast<long long>(blockIdx.x) * cap;
  int base = 0;   // sampled records before this pass (block-uniform)
  for (int j0 = 0; j0 < S && base <= cap; j0 += 4 * kSampleNT) {
    const int j = j0 + 4 * threadIdx.x;
    uint32_t bits = 0;
    if (j < S) {
      const uint32_t g = static_cast<uint32_t>(j) >> 2;
      const philox::U4 r = philox::philox4x32_10(philox::U4{g, 0u, word, kDpsgdSampleSite},
                                                 static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
      bits = static_cast<uint32_t>(r.x < thr) | (static_cast<uint32_t>(r.y < thr && j + 1 < S) << 1) |
             (static_cast<uint32_t>(r.z < thr && j + 2 < S) << 2) | (static_cast<uint32_t>(r.w < thr && j + 3 < S) << 3);
    }
    const int n = __popc(bits);
    int incl = n;   // inclusive warp scan
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (l >= o) incl += v;
    }
    if (l == 31) warp_tot[w] = incl;
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int k = 0; k < kSampleNT / 32; ++k) {
      const int t = warp_tot[k];
      before += k < w ? t : 0;
      total += t;
    }
    int pos = base + before + incl - n;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if ((bits >> e) & 1u) {
        if (pos < cap) out[pos] = j + e;
        ++pos;
      }
    }
    base += total;
    __syncthreads();   // warp_tot is rewritten by the next pass
  }
  const int kept = base < cap ? base : cap;
  for (int s = kept + threadIdx.x; s < cap; s += kSampleNT) out[s] = 0;
  if (threadIdx.x == 0) {
    count[blockIdx.x] = kept;
    if (base > cap) atomicAdd(overflow, 1);
  }
}

// ---------------------------------------------------------------- group norms
// one warp per example n: sq[n] = sum_c pg[n, c]^2 + pb[n, c]^2 over k_gn_bwd's own fp32 partials (lane l
// takes channels l, l + 32, ... in order, then the fixed butterfly)
__global__ void __launch_bounds__(32) k_pe_gn(const float* __restrict__ pg, const float* __restrict__ pb, int C,
                                              float* __restrict__ sq_out) {
  const long long base = static_cast<long long>(blockIdx.x) * C;
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += 32) s = fmaf(pg[base + c], pg[base + c], fmaf(pb[base + c], pb[base + c], s));
  s = warp_sum(s);
  if (threadIdx.x == 0) sq_out[blockIdx.x] = s;
}

// ---------------------------------------------------------------- deterministic split-K
// g[i] += sum_s ws[s * n + i], the slices in order: the fixed-order end of a split-K GEMM whose splits
// stored their partial tiles into their own slices
__global__ void k_sum_slices(const float* __restrict__ ws, int slices, long long n, float* __restrict__ g) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float t = ws[i];
    for (int k = 1; k < slices; ++k) t = so_add(t, ws[k * n + i]);
    g[i] = so_add(g[i], t);
  }
}

int grid_for(long long n, int per, int cap = 132 * 16) {
  long long b = (n + per - 1) / per;
  return static_cast<int>(b < 1 ? 1 : b > cap ? cap : b);
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace

cudaError_t dpsgd_pe_norm(const void* A, long long lda, int a_cols, const void* Bm, long long ldb, int b_cols,
                          int R, int n_ex, bool bias, float* out, cudaStream_t s, const DpsgdSegs* seg) {
  if (R < 1 || n_ex < 1 || a_cols < 1 || b_cols < 1 || (seg != nullptr && seg->cu == nullptr))
    return cudaErrorInvalidValue;
  const int vec_a = (lda % 8 == 0 && aligned16(A)) ? 1 : 0, vec_b = (ldb % 8 == 0 && aligned16(Bm)) ? 1 : 0;
  const int a_tiles = (a_cols + 63) / 64;
  const dim3 grid(dpsgd_norm_tiles(a_cols, b_cols, bias), n_ex);
  const bf16 *a = reinterpret_cast<const bf16*>(A), *b = reinterpret_cast<const bf16*>(Bm);
  (void)cudaGetLastError();
  if (seg == nullptr)
    k_pe_norm<<<grid, kNT, 0, s>>>(a, lda, a_cols, b, ldb, b_cols, R, n_ex, out, vec_a, vec_b, a_tiles,
                                   bias ? b_cols : -1);
  else
    k_packed_norm<<<grid, kNT, 0, s>>>(a, lda, a_cols, b, ldb, b_cols, n_ex, out, vec_a, vec_b, a_tiles,
                                       bias ? b_cols : -1, seg->cu, seg->rows);
  note_launch();
  return cudaGetLastError();
}

int dpsgd_norm_tiles(int a_cols, int b_cols, bool bias) {
  return ((a_cols + 63) / 64) * ((b_cols + (bias ? 1 : 0) + 63) / 64);
}

cudaError_t dpsgd_pe_gram(const DpsgdGram& a, int R, int n_ex, bool sym, float* out, cudaStream_t s,
                          const DpsgdSegs* seg) {
  const bool ok = a.mode == kGramDense    ? a.p1 != nullptr && a.p2 != nullptr && a.kp >= 1
                  : a.mode == kGramOneHot ? a.id1 != nullptr && a.id2 != nullptr
                  : a.mode == kGramGather ? a.p1 != nullptr && a.id2 != nullptr && a.kp >= 1
                                          : false;
  if (!ok || R < 1 || R > kMaxRowsR || n_ex < 1 || a.kq < 1 || a.q1 == nullptr || a.q2 == nullptr ||
      (seg != nullptr && seg->cu == nullptr))
    return cudaErrorInvalidValue;
  GramArgs g;
  g.p1 = reinterpret_cast<const bf16*>(a.p1);
  g.p2 = reinterpret_cast<const bf16*>(a.p2);
  g.ldp1 = a.ldp1;
  g.ldp2 = a.ldp2;
  g.kp = a.mode == kGramDense ? a.kp : 0;
  g.id1 = a.id1;
  g.id2 = a.id2;
  g.q1 = reinterpret_cast<const bf16*>(a.q1);
  g.q2 = reinterpret_cast<const bf16*>(a.q2);
  g.ldq1 = a.ldq1;
  g.ldq2 = a.ldq2;
  g.kq = a.kq;
  g.R = R;
  g.n_ex = n_ex;
  g.tiles = (R + 63) / 64;
  g.mode = a.mode;
  g.sym = sym ? 1 : 0;
  g.bias = a.bias;
  g.out = out;
  g.vec_p = (a.mode == kGramDense && a.ldp1 % 8 == 0 && a.ldp2 % 8 == 0 && aligned16(a.p1) && aligned16(a.p2)) ? 1 : 0;
  g.vec_q = (a.ldq1 % 8 == 0 && a.ldq2 % 8 == 0 && aligned16(a.q1) && aligned16(a.q2)) ? 1 : 0;
  (void)cudaGetLastError();
  if (seg == nullptr)
    k_pe_gram<<<dim3(dpsgd_gram_pairs(R, sym), n_ex), kNT, 0, s>>>(g);
  else
    k_packed_gram<<<dim3(dpsgd_gram_pairs(R, sym), n_ex), kNT, 0, s>>>(g, seg->cu, seg->rows);
  note_launch();
  return cudaGetLastError();
}

int dpsgd_gram_pairs(int R, bool sym) {
  const int t = (R + 63) / 64;
  return sym ? t * (t + 1) / 2 : t * t;
}

cudaError_t dpsgd_pe_ln(const void* dy, const void* x, int C, int R, int n_ex, const float* mean, const float* rstd,
                        float* sq_out, float* abs_out, cudaStream_t s, const DpsgdSegs* seg) {
  if (R < 1 || R > kMaxRowsR || n_ex < 1 || C < 1 || (seg != nullptr && seg->cu == nullptr))
    return cudaErrorInvalidValue;
  const bf16 *d = reinterpret_cast<const bf16*>(dy), *xx = reinterpret_cast<const bf16*>(x);
  (void)cudaGetLastError();
  if (seg == nullptr)
    k_pe_ln<<<n_ex, 256, 0, s>>>(d, xx, C, R, mean, rstd, sq_out, abs_out);
  else
    k_packed_ln<<<n_ex, 256, 0, s>>>(d, xx, C, mean, rstd, sq_out, abs_out, seg->cu, seg->rows);
  note_launch();
  return cudaGetLastError();
}

cudaError_t dpsgd_ln_release(const void* S, long long lds, const void* x, const float* mean, const float* rstd,
                             long long rows, int C, const float* c, int R, float* gg, float* gb, cudaStream_t s,
                             const DpsgdSegs* seg) {
  if (R < 1 || rows < 0 || C < 1 || (seg != nullptr && seg->seq == nullptr)) return cudaErrorInvalidValue;
  const bf16 *ss = reinterpret_cast<const bf16*>(S), *xx = reinterpret_cast<const bf16*>(x);
  (void)cudaGetLastError();
  if (seg == nullptr)
    k_ln_release<<<(C + 31) / 32, 512, 0, s>>>(ss, lds, xx, mean, rstd, rows, C, c, R, gg, gb);
  else
    k_packed_ln_release<<<(C + 31) / 32, 512, 0, s>>>(ss, lds, xx, mean, rstd, rows, C, c, gg, gb, seg->seq,
                                                      seg->n_ex);
  note_launch();
  return cudaGetLastError();
}

cudaError_t dpsgd_emb_release(const void* S, long long lds, int C, const int32_t* ids, int rows, int32_t* perm,
                              float* G, long long ldg, cudaStream_t s) {
  if (rows < 0 || C < 1) return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  (void)cudaGetLastError();
  k_id_rank<<<(rows + 255) / 256, 256, 0, s>>>(ids, rows, perm);
  note_launch();
  k_seg_release<<<rows, 128, 0, s>>>(reinterpret_cast<const bf16*>(S), lds, C, ids, perm, rows, G, ldg);
  note_launch();
  return cudaGetLastError();
}

cudaError_t dpsgd_pe_rows(const void* A, long long lda, int a_cols, const void* Bm, long long ldb, int b_cols,
                          int R, int n_ex, float bias, float* sq_out, float* abs_out, cudaStream_t s,
                          const DpsgdSegs* seg) {
  if (R < 1 || R > kMaxRowsAbs || n_ex < 1 || a_cols < 1 || b_cols < 0 ||
      (seg != nullptr && (seg->cu == nullptr || sq_out != nullptr)))
    return cudaErrorInvalidValue;
  const bf16 *a = reinterpret_cast<const bf16*>(A), *b = reinterpret_cast<const bf16*>(Bm);
  (void)cudaGetLastError();
  if (seg == nullptr)
    k_pe_rows<<<n_ex, 32 * (R < 8 ? R : 8), 0, s>>>(a, lda, a_cols, b, ldb, b_cols, R, bias, sq_out, abs_out);
  else   // the warp count does not change the bits (k_pe_rows): R is the longest example's rows
    k_packed_rows<<<n_ex, 32 * (R < 8 ? R : 8), 0, s>>>(a, lda, a_cols, b, ldb, b_cols, bias, abs_out, seg->cu,
                                                        seg->rows);
  note_launch();
  return cudaGetLastError();
}

cudaError_t dpsgd_clip(const float* sq, int n_sq, const float* ab, int n_ab, const float* kap, int n_ex, float bsz,
                       float clip, float* c, int* dropped, const int* n_valid, cudaStream_t s) {
  if (n_ex < 1 || n_sq < 0 || n_ab < 0) return cudaErrorInvalidValue;
  (void)cudaGetLastError();
  k_dpsgd_clip<<<(n_ex + 127) / 128, 128, 0, s>>>(sq, n_sq, ab, n_ab, kap, n_ex, bsz, clip, c, dropped, n_valid);
  note_launch();
  return cudaGetLastError();
}

cudaError_t dpsgd_scale_rows(const void* X, long long ldx, void* out, long long ldo, long long rows, int cols,
                             const float* c, int R, bool mask_only, cudaStream_t s, const DpsgdSegs* seg) {
  if (R < 1 || rows < 0 || cols < 1 || (seg != nullptr && seg->seq == nullptr)) return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  const bf16* xx = reinterpret_cast<const bf16*>(X);
  bf16* o = reinterpret_cast<bf16*>(out);
  (void)cudaGetLastError();
  if (seg == nullptr)
    k_scale_rows<<<grid_for(rows * cols, 256), 256, 0, s>>>(xx, ldx, o, ldo, rows, cols, c, R, mask_only ? 1 : 0);
  else
    k_packed_scale_rows<<<grid_for(rows * cols, 256), 256, 0, s>>>(xx, ldx, o, ldo, rows, cols, c, mask_only ? 1 : 0,
                                                                   seg->seq, seg->n_ex);
  note_launch();
  return cudaGetLastError();
}

cudaError_t dpsgd_colsum(const void* X, long long ld, long long rows, int cols, float* g, cudaStream_t s) {
  if (rows < 0 || cols < 1) return cudaErrorInvalidValue;
  (void)cudaGetLastError();
  k_colsum_fixed<<<(cols + 31) / 32, 512, 0, s>>>(reinterpret_cast<const bf16*>(X), ld, rows, cols, g);
  note_launch();
  return cudaGetLastError();
}

cudaError_t dpsgd_noise(float* g, long long P, uint64_t seed, const int32_t* step, uint32_t add, float sigma,
                        cudaStream_t s) {
  if (P < 0) return cudaErrorInvalidValue;
  if (P == 0) return cudaSuccess;
  (void)cudaGetLastError();
  k_dpsgd_noise<<<grid_for((P + 3) / 4, 256), 256, 0, s>>>(g, P, seed, step, add, sigma);
  note_launch();
  return cudaGetLastError();
}

cudaError_t dpsgd_poisson_sample(uint64_t seed, const int32_t* step, int steps, int S, uint32_t thr, int cap,
                                 int32_t* idx, int32_t* count, int32_t* overflow, cudaStream_t s) {
  if (steps < 1 || S < 1 || thr == 0u || cap < 1 || cap > S) return cudaErrorInvalidValue;
  (void)cudaGetLastError();
  k_dpsgd_poisson_sample<<<steps, kSampleNT, 0, s>>>(seed, step, S, thr, cap, idx, count, overflow);
  note_launch();
  return cudaGetLastError();
}

cudaError_t dpsgd_pe_gn(const float* pg, const float* pb, int n_ex, int C, float* sq_out, cudaStream_t s) {
  if (n_ex < 1 || C < 1) return cudaErrorInvalidValue;
  (void)cudaGetLastError();
  k_pe_gn<<<n_ex, 32, 0, s>>>(pg, pb, C, sq_out);
  note_launch();
  return cudaGetLastError();
}

cudaError_t dpsgd_sum_slices(const float* ws, int slices, long long n, float* g, cudaStream_t s) {
  if (slices < 1 || n < 0) return cudaErrorInvalidValue;
  if (n == 0) return cudaSuccess;
  (void)cudaGetLastError();
  k_sum_slices<<<grid_for(n, 256), 256, 0, s>>>(ws, slices, n, g);
  note_launch();
  return cudaGetLastError();
}

cudaError_t dpsgd_patch_rows(const void* dz, long long ldz, int Cout, const void* x, int N, int H, int W, int C,
                             int OH, int OW, int KH, int KW, int stride, int pad, float bias, float* abs_out,
                             cudaStream_t s) {
  const int R = OH * OW;
  if (N < 1 || R < 1 || R > kMaxRowsAbs || Cout < 1 || C < 1 || KH < 1 || KW < 1 || stride < 1 || pad < 0)
    return cudaErrorInvalidValue;
  (void)cudaGetLastError();
  k_patch_rows<<<N, 32 * (R < 8 ? R : 8), 0, s>>>(reinterpret_cast<const bf16*>(dz), ldz, Cout,
                                                  reinterpret_cast<const bf16*>(x), H, W, C, OH, OW, KH, KW, stride,
                                                  pad, bias, abs_out);
  note_launch();
  return cudaGetLastError();
}

}  // namespace bflc
