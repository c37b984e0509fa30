// DP-SGD (Abadi et al. 2016) with book-keeping clipping (ops/dpsgd.py): per-example gradient norms,
// certified clip factors, per-example row scaling, deterministic bias column sums and the client's
// Gaussian noise.
//
// A weight gradient over B examples of R rows each is G = sum_n A_n^T Bm_n, A_n / Bm_n the n-th R-row
// blocks of A [B*R, a] and Bm [B*R, b].  The per-example part ||A_n^T Bm_n||_F^2 never materialises:
// k_pe_norm keeps one 64 x 64 product tile of it in wgmma accumulators (the wide side a as the M
// dimension, the narrow side b <= 64 as N, the example's tokens as K, both operands MN-major, read
// straight from the row-major activations) and its epilogue squares and reduces the tile to one fp32
// partial per (tile, example).  R = 1 sites (whole-row layers) use the identity
// ||dz x^T||^2 + ||dz||^2 = ||dz||^2 (||x||^2 + 1) in k_pe_rows instead.  Every sum runs in a fixed
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

// the 64-token chunk starting at token t0 of example rows [row0, row0 + R): 512 16-byte pieces per
// operand, four per thread; piece (t, c) is token t, columns 8c .. 8c + 7 of the tile
__device__ __forceinline__ void fetch(uint4 (&ra)[4], uint4 (&rb)[4], const bf16* __restrict__ A, long long lda,
                                      int a_cols, const bf16* __restrict__ Bm, long long ldb, int b_cols,
                                      long long row0, int R, int t0, int col0, bool vec_a, bool vec_b) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = threadIdx.x + kNT * i, t = idx >> 3, c = idx & 7;
    const bool ok = t0 + t < R;
    ra[i] = load8(A, lda, row0 + t0 + t, ok, col0 + 8 * c, a_cols, vec_a);
    rb[i] = load8(Bm, ldb, row0 + t0 + t, ok, 8 * c, b_cols, vec_b);
  }
}

// grid (ceil(a / 64), B): out[tile * B + n] = sum over the tile's 64 x 64 entries of (A_n^T Bm_n)^2
__global__ void __launch_bounds__(kNT) k_pe_norm(const bf16* __restrict__ A, long long lda, int a_cols,
                                                 const bf16* __restrict__ Bm, long long ldb, int b_cols, int R,
                                                 int n_ex, float* __restrict__ out, int vec_a, int vec_b) {
  // MN-major 128B-swizzled operand tiles [64 tokens][64 columns]: token t is the 128-byte row t, its
  // 16-byte piece c sits at piece c ^ (t & 7)
  __shared__ __align__(1024) uint8_t sm[2 * 8192];
  __shared__ float red[4];
  const int n = blockIdx.y, col0 = blockIdx.x * 64;
  const long long row0 = static_cast<long long>(n) * R;
  const uint32_t sa = ptx::smem_u32(sm), sb = sa + 8192u;
  float d[32];
  wg::zero(d);
  uint4 ra[4], rb[4];
  fetch(ra, rb, A, lda, a_cols, Bm, ldb, b_cols, row0, R, 0, col0, vec_a != 0, vec_b != 0);
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
      fetch(ra, rb, A, lda, a_cols, Bm, ldb, b_cols, row0, R, t0 + 64, col0, vec_a != 0, vec_b != 0);
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

// one block of min(R, 8) warps per example n.  Row t of the example gets ra_t = ||A_t||^2 and
// rb_t = ||Bm_t||^2 + bias; abs_out[n] = sum_t sqrt(ra_t) sqrt(rb_t) in token order, and for R = 1
// sq_out[n] = ra_0 rb_0 (the squared norm of the row's weight-and-bias gradient)
constexpr int kMaxRowsR = 512;
__global__ void __launch_bounds__(256) k_pe_rows(const bf16* __restrict__ A, long long lda, int a_cols,
                                                 const bf16* __restrict__ Bm, long long ldb, int b_cols, int R,
                                                 float bias, float* __restrict__ sq_out, float* __restrict__ abs_out) {
  __shared__ float term[kMaxRowsR];
  const int n = blockIdx.x, w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int t = w; t < R; t += nw) {
    const long long row = static_cast<long long>(n) * R + t;
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

// c[n] from the sites' partials sq [n_sq][B] and abs [n_ab][B] (DESIGN.md, "DP-SGD"):
//   norm = sqrt(sum sq), bound = (B norm) (1 + gamma) + (B abs) (u + gamma),
//   c = 0 for a non-finite bound (the example is dropped and counted), else 1 if bound <= C, else C / bound
constexpr float kOnePlusGamma = 1.0009765625f;   // 1 + 2^-10
constexpr float kUPlusGamma = 0.0048828125f;     // 2^-8 + 2^-10
__global__ void k_dpsgd_clip(const float* __restrict__ sq, int n_sq, const float* __restrict__ ab, int n_ab,
                             int n_ex, float bsz, float clip, float* __restrict__ c, int* __restrict__ dropped) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_ex) return;
  float s = 0.f, a = 0.f;
  for (int i = 0; i < n_sq; ++i) s = so_add(s, sq[static_cast<long long>(i) * n_ex + n]);
  for (int i = 0; i < n_ab; ++i) a = so_add(a, ab[static_cast<long long>(i) * n_ex + n]);
  const float bound = so_add(so_mul(so_mul(so_sqrt(s), bsz), kOnePlusGamma), so_mul(so_mul(a, bsz), kUPlusGamma));
  if ((dp_bits(bound) & 0x7F800000u) == 0x7F800000u) {   // inf or NaN
    c[n] = 0.f;
    atomicAdd(dropped, 1);
  } else {
    c[n] = dp_scale(bound, clip);
  }
}

// out[r, j] = bf16(X[r, j] * c[r / R]) (mask_only: X[r, j] unscaled), and exactly +0 where c[r / R] is 0:
// a dropped example's rows may hold NaN or inf, which a product with 0 would keep
__global__ void k_scale_rows(const bf16* __restrict__ X, long long ldx, bf16* __restrict__ out, long long ldo,
                             long long rows, int cols, const float* __restrict__ c, int R, int mask_only) {
  const long long total = rows * cols;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / cols;
    const int j = static_cast<int>(i - r * cols);
    const float cr = c[r / R];
    const bf16 x = X[r * ldx + j];
    out[r * ldo + j] = (dp_bits(cr) & 0x7FFFFFFFu) == 0u ? __float2bfloat16_rn(0.f)
                       : mask_only                        ? x
                                                          : __float2bfloat16_rn(so_mul(__bfloat162float(x), cr));
  }
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

int grid_for(long long n, int per, int cap = 132 * 16) {
  long long b = (n + per - 1) / per;
  return static_cast<int>(b < 1 ? 1 : b > cap ? cap : b);
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace

cudaError_t dpsgd_pe_norm(const void* A, long long lda, int a_cols, const void* Bm, long long ldb, int b_cols,
                          int R, int n_ex, float* out, cudaStream_t s) {
  if (R < 1 || n_ex < 1 || a_cols < 1 || b_cols < 1 || b_cols > 64) return cudaErrorInvalidValue;
  const int vec_a = (lda % 8 == 0 && aligned16(A)) ? 1 : 0, vec_b = (ldb % 8 == 0 && aligned16(Bm)) ? 1 : 0;
  (void)cudaGetLastError();
  k_pe_norm<<<dim3((a_cols + 63) / 64, n_ex), kNT, 0, s>>>(
      reinterpret_cast<const bf16*>(A), lda, a_cols, reinterpret_cast<const bf16*>(Bm), ldb, b_cols, R, n_ex, out,
      vec_a, vec_b);
  note_launch();
  return cudaGetLastError();
}

cudaError_t dpsgd_pe_rows(const void* A, long long lda, int a_cols, const void* Bm, long long ldb, int b_cols,
                          int R, int n_ex, float bias, float* sq_out, float* abs_out, cudaStream_t s) {
  if (R < 1 || R > kMaxRowsR || n_ex < 1 || a_cols < 1 || b_cols < 0) return cudaErrorInvalidValue;
  (void)cudaGetLastError();
  k_pe_rows<<<n_ex, 32 * (R < 8 ? R : 8), 0, s>>>(reinterpret_cast<const bf16*>(A), lda, a_cols,
                                                  reinterpret_cast<const bf16*>(Bm), ldb, b_cols, R, bias, sq_out,
                                                  abs_out);
  note_launch();
  return cudaGetLastError();
}

cudaError_t dpsgd_clip(const float* sq, int n_sq, const float* ab, int n_ab, int n_ex, float bsz, float clip,
                       float* c, int* dropped, cudaStream_t s) {
  if (n_ex < 1 || n_sq < 0 || n_ab < 0) return cudaErrorInvalidValue;
  (void)cudaGetLastError();
  k_dpsgd_clip<<<(n_ex + 127) / 128, 128, 0, s>>>(sq, n_sq, ab, n_ab, n_ex, bsz, clip, c, dropped);
  note_launch();
  return cudaGetLastError();
}

cudaError_t dpsgd_scale_rows(const void* X, long long ldx, void* out, long long ldo, long long rows, int cols,
                             const float* c, int R, bool mask_only, cudaStream_t s) {
  if (R < 1 || rows < 0 || cols < 1) return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  (void)cudaGetLastError();
  k_scale_rows<<<grid_for(rows * cols, 256), 256, 0, s>>>(reinterpret_cast<const bf16*>(X), ldx,
                                                         reinterpret_cast<bf16*>(out), ldo, rows, cols, c, R,
                                                         mask_only ? 1 : 0);
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

}  // namespace bflc
