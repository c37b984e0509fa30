// Fused multi-head self-attention, head_dim = 64.  Unmasked seq_len = 128 (BERT-base, BASELINE.json
// config #5) runs the kernels right below; any other seq_len % 64 == 0 up to 512, or a key-padding
// mask, runs the tiled kernels further down ("variable length, masked").
//
// seq_len = 128: one CTA per (batch, head) = one warpgroup, every GEMM a Hopper wgmma with register
// accumulators, the S x S score / probability matrix never leaves the SM.  Each GEMM runs as two
// m64 halves (query rows, or key rows for dK / dV) so that at most two 64 x 128 fp32 fragments
// are live at a time.
//
//   forward   S = Q K^T  ->  row softmax on the fragments (a row is spread over 4 lanes)  ->  P as bf16
//             into a 128B-swizzled smem A-operand tile  ->  O = P V (V as MN-major B operand)  ->
//             O / rowsum -> global.  Saves lse[row] = max + log(sum) for the backward pass.
//   backward  recompute S and P = exp(S - lse); dP = dO V^T; dS = P (dP - delta) with
//             delta = rowsum(dO * O); then three GEMMs out of smem-resident P / dS:
//             dQ = dS K,  dK = dS^T Q,  dV = P^T dO  (P and dS written once K-major and once
//             MN-major: the same rows, two block arrangements).
//
// q, k, v, o and their gradients are [B*S, H*D] row-major matrices (the projection outputs as
// they are): head h of batch b is the TMA box {64 columns from h*64, 128 rows from b*128}, so no
// head transpose exists anywhere.  The unfused path this replaces (ops/nn.py, round 1) ran two
// batched GEMMs, a softmax kernel and four transposes and wrote the S x S probabilities to HBM.
// No reference counterpart (the reference model is a 5x2 softmax regression, python-sdk/main.py:113-120).
#include <cuda_bf16.h>

#include <type_traits>

#include "bflc_kernels.h"
#include "epi_common.cuh"
#include "launch.cuh"
#include "philox.hpp"
#include "sm100_ptx.cuh"
#include "wgmma.cuh"

namespace bflc {

namespace {

__device__ __forceinline__ uint32_t pack2(float a, float b) { return epi::pack_bf16x2(a, b); }

constexpr int kS = 128, kD = 64;
constexpr int kTile = kS * 128;          // one [128 rows x 64 bf16] operand tile: 16 KB
constexpr int kThreads = 128;            // one warpgroup
constexpr float kLog2e = 1.4426950408889634f;

struct AttnP {
  int H; long long ld; float scale;
  __nv_bfloat16* o; float* lse;                     // forward outputs ([B*S, ld], [B*H*S])
  const __nv_bfloat16* o_in; const __nv_bfloat16* dout_g;   // backward: saved O, dO (for delta)
  __nv_bfloat16* dq; __nv_bfloat16* dk; __nv_bfloat16* dv;
};

// bf16 pair (col, col + 1) of row m of a 128 x 128 matrix kept as 128B-swizzled operand tiles:
//   K-major (K = column):      tile col / 64, row m
//   MN-major (K = row index):  K-block m / 64, M-chunk col / 64, row m % 64
__device__ __forceinline__ void put2_kmaj(uint8_t* base, int m, int col, float a, float b) {
  uint8_t* t = base + (col >> 6) * kTile + m * 128;
  *reinterpret_cast<uint32_t*>(t + ((((col & 63) >> 3) ^ (m & 7)) << 4) + (col & 7) * 2) = pack2(a, b);
}
__device__ __forceinline__ void put2_mnmaj(uint8_t* base, int m, int col, float a, float b) {
  uint8_t* t = base + (m >> 6) * kTile + (col >> 6) * 8192 + (m & 63) * 128;
  *reinterpret_cast<uint32_t*>(t + ((((col & 63) >> 3) ^ (m & 7)) << 4) + (col & 7) * 2) = pack2(a, b);
}
// rows 64h.. of [128 x 128] = A (K-major, K = 64) . B^T (K-major, 128 rows)
__device__ __forceinline__ void mma_s(float (&d)[64], uint32_t a_addr, uint32_t b_addr, int h) {
#pragma unroll
  for (uint32_t k = 0; k < 4; ++k)
    wg::mma_bf16<128, 0, 0>(d, wg::desc(a_addr + h * 8192u + k * 32u, 16), wg::desc(b_addr + k * 32u, 16), k > 0);
}
// rows 64h.. of [128 x 64] = A (K-major [128 x 128] as two 64-wide K tiles) . B (MN-major [128 K][64])
__device__ __forceinline__ void mma_kmaj_bmn(float (&d)[32], uint32_t a_addr, uint32_t b_addr, int h) {
#pragma unroll
  for (uint32_t ks = 0; ks < 8; ++ks)
    wg::mma_bf16<64, 0, 1>(d, wg::desc(a_addr + (ks >> 2) * kTile + h * 8192u + (ks & 3u) * 32u, 16),
                           wg::desc(b_addr + ks * 2048u, 8192), ks > 0);
}
// rows 64h.. of [128 x 64] = A^T (A MN-major: K-block kb = two 64-wide M-chunks) . B (MN-major)
__device__ __forceinline__ void mma_amn_bmn(float (&d)[32], uint32_t a_addr, uint32_t b_addr, int h) {
#pragma unroll
  for (uint32_t ks = 0; ks < 8; ++ks)
    wg::mma_bf16<64, 1, 1>(d, wg::desc(a_addr + (ks >> 2) * kTile + h * 8192u + (ks & 3u) * 2048u, 8192),
                           wg::desc(b_addr + ks * 2048u, 8192), ks > 0);
}
template <int R>
__device__ __forceinline__ void run_sync(float (&d)[R]) {
  wg::commit();
  wg::wait<0>();
  wg::reg_fence(d);
}
// 64-column fragment (rows row0 + lane/4 [+8]) -> bf16 global rows, scaled by mul0 / mul1
__device__ __forceinline__ void store_frag64(const float (&d)[32], __nv_bfloat16* base, long long ld, int row0,
                                             float mul0, float mul1) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int hi = (i >> 1) & 1;
    const int r = row0 + (lane >> 2) + 8 * hi, c = wg::frag_col(i, lane);
    const float m = hi ? mul1 : mul0;
    *reinterpret_cast<uint32_t*>(base + r * ld + c) = pack2(d[i] * m, d[i + 1] * m);
  }
}
// store_frag64 for rows < row_end only (packed sequences: the next rows belong to another sequence)
__device__ __forceinline__ void store_frag64_rows(const float (&d)[32], __nv_bfloat16* base, long long ld, int row0,
                                                  float mul0, float mul1, int row_end) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int hi = (i >> 1) & 1;
    const int r = row0 + (lane >> 2) + 8 * hi, c = wg::frag_col(i, lane);
    const float m = hi ? mul1 : mul0;
    if (r < row_end) *reinterpret_cast<uint32_t*>(base + r * ld + c) = pack2(d[i] * m, d[i + 1] * m);
  }
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// ------------------------------------------------------------------------------------ forward
constexpr int kFwdSmem = 3 * kTile + 2 * kTile + 256 + 1024;

__global__ void __launch_bounds__(kThreads, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttnP p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem; uint8_t* sK = smem + kTile; uint8_t* sV = smem + 2 * kTile; uint8_t* sP = smem + 3 * kTile;
  uint64_t* bar_in = reinterpret_cast<uint64_t*>(smem + 5 * kTile);
  ptx::pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x / p.H, h = blockIdx.x % p.H;
  if (threadIdx.x == 0) {
    ptx::mbar_init(bar_in, 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  ptx::pdl_wait();
  if (threadIdx.x == 0) {
    ptx::mbar_expect_tx(bar_in, 3 * kTile);
    ptx::tma_load_3d(sQ, &tmQ, bar_in, h * kD, b * kS, 0);
    ptx::tma_load_3d(sK, &tmK, bar_in, h * kD, b * kS, 0);
    ptx::tma_load_3d(sV, &tmV, bar_in, h * kD, b * kS, 0);
  }
  ptx::mbar_wait(bar_in, 0);
  const float sc = p.scale * kLog2e;
  float inv[2][2];
#pragma unroll 1
  for (int half = 0; half < 2; ++half) {
    float s[64];
    wg::fence();
    mma_s(s, ptx::smem_u32(sQ), ptx::smem_u32(sK), half);   // S = Q K^T
    run_sync(s);
    const int r0 = 64 * half + 16 * warp + (lane >> 2);   // this thread's rows r0 and r0 + 8
    float mx[2] = {-INFINITY, -INFINITY}, sum[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 64; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
    mx[0] = quad_max(mx[0]); mx[1] = quad_max(mx[1]);
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      s[i] = exp2f((s[i] - mx[(i >> 1) & 1]) * sc);
      sum[(i >> 1) & 1] += s[i];
    }
    sum[0] = quad_sum(sum[0]); sum[1] = quad_sum(sum[1]);
#pragma unroll
    for (int i = 0; i < 64; i += 2) put2_kmaj(sP, r0 + 8 * ((i >> 1) & 1), wg::frag_col(i, lane), s[i], s[i + 1]);
    if ((lane & 3) == 0) {
#pragma unroll
      for (int e = 0; e < 2; ++e)
        p.lse[static_cast<long long>(blockIdx.x) * kS + r0 + 8 * e] = mx[e] * p.scale + __logf(sum[e]);
    }
    inv[half][0] = 1.f / sum[0]; inv[half][1] = 1.f / sum[1];
  }
  ptx::fence_proxy_async_smem();   // P (generic stores) -> wgmma operand reads
  __syncthreads();
  const long long gbase = static_cast<long long>(b) * kS * p.ld + h * kD;
#pragma unroll 1
  for (int half = 0; half < 2; ++half) {
    float o[32];
    wg::fence();
    mma_kmaj_bmn(o, ptx::smem_u32(sP), ptx::smem_u32(sV), half);   // O = P V
    run_sync(o);
    store_frag64(o, p.o + gbase, p.ld, 64 * half + 16 * warp, inv[half][0], inv[half][1]);
  }
}

// ----------------------------------------------------------------------------------- backward
constexpr int kBwdSmem = 4 * kTile + 3 * 2 * kTile + 256 + 1024;

__global__ void __launch_bounds__(kThreads, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                const AttnP p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem; uint8_t* sK = smem + kTile; uint8_t* sV = smem + 2 * kTile; uint8_t* sDO = smem + 3 * kTile;
  uint8_t* sPt = smem + 4 * kTile;        // P, MN-major arrangement (A of dV = P^T dO)
  uint8_t* sDSk = smem + 6 * kTile;       // dS, K-major (A of dQ = dS K)
  uint8_t* sDSt = smem + 8 * kTile;       // dS, MN-major (A of dK = dS^T Q)
  uint64_t* bar_in = reinterpret_cast<uint64_t*>(smem + 10 * kTile);
  ptx::pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x / p.H, h = blockIdx.x % p.H;
  if (threadIdx.x == 0) {
    ptx::mbar_init(bar_in, 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  ptx::pdl_wait();
  if (threadIdx.x == 0) {
    ptx::mbar_expect_tx(bar_in, 4 * kTile);
    ptx::tma_load_3d(sQ, &tmQ, bar_in, h * kD, b * kS, 0);
    ptx::tma_load_3d(sK, &tmK, bar_in, h * kD, b * kS, 0);
    ptx::tma_load_3d(sV, &tmV, bar_in, h * kD, b * kS, 0);
    ptx::tma_load_3d(sDO, &tmDO, bar_in, h * kD, b * kS, 0);
  }
  const float sc = p.scale * kLog2e;
#pragma unroll 1
  for (int half = 0; half < 2; ++half) {
    const int r0 = 64 * half + 16 * warp + (lane >> 2);
    // delta = rowsum(dO * O) = rowsum(dP * P) of rows r0, r0 + 8, and their lse, from global
    float delta[2] = {0.f, 0.f}, lse2[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const long long grow = static_cast<long long>(b) * kS + r0 + 8 * e;
      const uint4* o4 = reinterpret_cast<const uint4*>(p.o_in + grow * p.ld + h * kD);
      const uint4* d4 = reinterpret_cast<const uint4*>(p.dout_g + grow * p.ld + h * kD);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint4 a = o4[j], c = d4[j];
        const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, cw[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 fa = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&aw[q]));
          const float2 fc = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&cw[q]));
          delta[e] += fa.x * fc.x + fa.y * fc.y;
        }
      }
      lse2[e] = p.lse[static_cast<long long>(blockIdx.x) * kS + r0 + 8 * e] * kLog2e;
    }
    if (half == 0) ptx::mbar_wait(bar_in, 0);
    float s[64], dp[64];
    wg::fence();
    mma_s(s, ptx::smem_u32(sQ), ptx::smem_u32(sK), half);      // S  = Q K^T
    mma_s(dp, ptx::smem_u32(sDO), ptx::smem_u32(sV), half);    // dP = dO V^T
    wg::commit();
    wg::wait<0>();
    wg::reg_fence(s);
    wg::reg_fence(dp);
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int e = (i >> 1) & 1, m = r0 + 8 * e, col = wg::frag_col(i, lane);
      const float p0 = exp2f(s[i] * sc - lse2[e]), p1 = exp2f(s[i + 1] * sc - lse2[e]);
      const float d0 = p0 * (dp[i] - delta[e]) * p.scale, d1 = p1 * (dp[i + 1] - delta[e]) * p.scale;
      put2_mnmaj(sPt, m, col, p0, p1);
      put2_kmaj(sDSk, m, col, d0, d1);
      put2_mnmaj(sDSt, m, col, d0, d1);
    }
  }
  ptx::fence_proxy_async_smem();
  __syncthreads();
  const long long gbase = static_cast<long long>(b) * kS * p.ld + h * kD;
#pragma unroll 1
  for (int half = 0; half < 2; ++half) {
    // accumulator row m of dQ is query row m; of dK / dV it is key row m
    const int row0 = 64 * half + 16 * warp;
    float acc[32];
    wg::fence();
    mma_kmaj_bmn(acc, ptx::smem_u32(sDSk), ptx::smem_u32(sK), half);   // dQ = dS K
    run_sync(acc);
    store_frag64(acc, p.dq + gbase, p.ld, row0, 1.f, 1.f);
    wg::fence();
    mma_amn_bmn(acc, ptx::smem_u32(sDSt), ptx::smem_u32(sQ), half);    // dK = dS^T Q
    run_sync(acc);
    store_frag64(acc, p.dk + gbase, p.ld, row0, 1.f, 1.f);
    wg::fence();
    mma_amn_bmn(acc, ptx::smem_u32(sPt), ptx::smem_u32(sDO), half);    // dV = P^T dO
    run_sync(acc);
    store_frag64(acc, p.dv + gbase, p.ld, row0, 1.f, 1.f);
  }
}

// ====================================================================== variable length, masked
// Tiled kernels for S % 64 == 0, 64 <= S <= 512 with a right-padding key mask: query row i of
// sequence b attends to keys j < len_b, len_b = min(lengths[b], S) (lengths == nullptr: S).
// Work is counted in 64-row blocks, and no key block at or beyond len_b is ever loaded.
//   forward  one CTA per (b, h, 128-query block).  MMA warpgroups 0 / 1 own 64 query rows each;
//            warp 8 streams K / V blocks through a kVStages-deep TMA + mbarrier ring.  Online
//            softmax: running max m and sum l per row; lse = m * scale + log(l) is saved.
//   dQ       one CTA per (b, h, 128-query block), the same roles, looping over the valid K / V
//            blocks; it also writes delta = rowsum(dO * O) of its rows for the dK / dV kernel.
//   dK / dV  one CTA per (b, h, 64-key block): one MMA warpgroup with the keys as the M rows
//            (S^T = K Q^T, dP^T = V dO^T) and producer warp 4 streaming Q / dO blocks plus their
//            lse / delta rows.  It loops over every query block: padded query rows are computed,
//            as scaled_dot_product_attention computes them, and so carry gradient.  A key block
//            at or beyond len_b writes zero rows and loads nothing.
// Every output element is written once by one thread (no atomics), so results are
// bit-reproducible.  len_b <= 0 gives zero outputs and gradients (no NaN: l = 0 is never divided).
//
// Packed mode (kPacked = true): the real tokens of all sequences are concatenated, q ... dv are
// [T, ld] and sequence b is rows [cu[b], cu[b+1]) (cu_seqlens, int32 [B+1]).  S is max_seqlen
// rounded up to 64; it sizes the grid and the [B*H, S] lse / delta workspaces, which stay indexed
// by the in-sequence row.  len_b = cu[b+1] - cu[b], clamped to S and to the rows before T.
// Differences from the padded mode:
//   * a CTA whose block starts at or past len_b returns before any TMA and writes nothing (there
//     is no padding to zero); the CTAs that work count their live warpgroups from len_b;
//   * TMA boxes start at row cu[b] + 64 * block on maps of T rows: past T they zero-fill, and rows
//     past len_b inside T belong to the next sequence, so besides the masked keys the dK / dV
//     kernel also masks query columns >= len_b (P = dS = 0, by select);
//   * dK / dV loops over the query blocks that hold real rows only;
//   * every store of o, dq, dk, dv, and the dQ kernel's reads of o / dO for delta, are limited to
//     rows < len_b (delta = 0 past it).
//
// Causal mode (kCausal: padded mode without lengths; kernels attn_causal_{fwd,dq,dkv}): query row i attends to keys j <= i.  Key
// blocks above the diagonal are never loaded or multiplied:
//   * forward / dQ: warpgroup g of query block qb (64-row block 2 qb + g) stops after its diagonal
//     key block 2 qb + g, and the producer streams blocks 0 .. 2 qb + live - 1, up to the last live
//     warpgroup's diagonal.  empty[s] still counts 4 * live arrivals.  Warpgroup 0 skips only the
//     producer's last block (2 qb + 1), whose stage the producer never waits on again: it waits on
//     empty[s] of block j - kVStages before loading block j, and every block below 2 qb + 1 is
//     consumed, and arrived on, by every live warpgroup.  Warpgroup 0 must not arrive for the
//     skipped block either: it may still be a phase ahead of warpgroup 1 on that stage, and an early
//     arrival would complete the phase of block 2 qb + 1 - kVStages while warpgroup 1 still reads it;
//   * dK / dV: key block kb starts its query loop at query block kb;
//   * only the diagonal block masks single elements: S = -inf before the exp (forward), P = dS = 0
//     (backward), for key column > query row.
constexpr int kVB = 64;                      // rows of one streamed block
constexpr int kVQ = 128;                     // query rows of a forward / dQ CTA
constexpr int kVTile = kVB * 128;            // one [64 rows x 64 bf16] operand tile: 8 KB
constexpr int kVStages = 4;
constexpr int kVThreads = 288;               // warps 0-7: two MMA warpgroups, warp 8: producer
constexpr int kVThreadsKV = 160;             // warps 0-3: one MMA warpgroup, warp 4: producer
constexpr int kVMaxS = 512;

struct VarP {
  int S, H; long long ld; float scale;
  const int32_t* lengths;
  __nv_bfloat16* o; float* lse;
  const __nv_bfloat16* o_in; const __nv_bfloat16* dout_g; float* delta;
  __nv_bfloat16* dq; __nv_bfloat16* dk; __nv_bfloat16* dv;
  const int32_t* cu; int T;                         // packed mode: cu_seqlens [B+1], total rows
};
// The dropout instantiations (kDrop) take these instead; the others keep VarP as it is.
// step = *drop_step + drop_add, read after the dependency wait (philox.hpp).
struct VarPDrop : VarP {
  const int32_t* drop_step; int drop_add; uint32_t seed_lo, seed_hi, site, thr; float dscale;
};
template <bool kDrop>
using VarArgs = typename std::conditional<kDrop, VarPDrop, VarP>::type;

__device__ __forceinline__ uint8_t* align1024(uint8_t* p) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~static_cast<uintptr_t>(1023));
}
__device__ __forceinline__ int valid_len(const VarP& p, int b) { return p.lengths ? min(p.lengths[b], p.S) : p.S; }
// packed mode: rows of sequence b that lie in [0, T), at most S (a bad cu value cannot walk off the buffers)
__device__ __forceinline__ int packed_len(const VarP& p, int b) {
  const int r0 = p.cu[b];
  return r0 < 0 ? 0 : min(min(p.cu[b + 1], p.T) - r0, p.S);
}
__device__ __forceinline__ int key_blocks(int len) { return len > 0 ? (len + kVB - 1) / kVB : 0; }
// query warpgroups of a 128-row block that lie inside the sequence (1 for the last block of S = 64 (mod 128))
__device__ __forceinline__ int live_groups(int S, int qb) { return min(2, (S - qb * kVQ) / kVB); }
// barrier among the 128 threads of one warpgroup (ids 1, 2; 0 is __syncthreads)
__device__ __forceinline__ void wg_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// [64 x 64] = A (K-major [64 x 64]) . B^T (K-major [64 x 64])
__device__ __forceinline__ void mma_nt64(float (&d)[32], uint32_t a, uint32_t b) {
#pragma unroll
  for (uint32_t k = 0; k < 4; ++k)
    wg::mma_bf16<64, 0, 0>(d, wg::desc(a + k * 32u, 16), wg::desc(b + k * 32u, 16), k > 0);
}
// d += A (K-major [64 x 64]) . B (MN-major: 64 K rows of 64)
__device__ __forceinline__ void mma_nn64(float (&d)[32], uint32_t a, uint32_t b) {
#pragma unroll
  for (uint32_t k = 0; k < 4; ++k)
    wg::mma_bf16<64, 0, 1>(d, wg::desc(a + k * 32u, 16), wg::desc(b + k * 2048u, 8192), 1u);
}
template <int R>
__device__ __forceinline__ void run_sync2(float (&a)[R], float (&b)[R]) {
  wg::commit();
  wg::wait<0>();
  wg::reg_fence(a);
  wg::reg_fence(b);
}

// ---- attention-probability dropout (kDrop).  Every warp draws the keep bits of exactly the
// 16 x 64 (rows x columns of its accumulator) elements it owns: 128 Philox calls of 8 columns, 4 per
// lane, into a private 128-byte smem mask, then each lane reads back its own bits (__syncwarp in
// between; the __syncwarp that ends every block iteration orders the next draw after the reads).
__device__ __forceinline__ philox::Drop drop_of(const VarPDrop& p) {
  return philox::Drop{p.seed_lo, p.seed_hi, static_cast<uint32_t>(*p.drop_step + p.drop_add), p.site, p.thr,
                      p.dscale};
}
// Forward / dQ layout (accumulator rows = query rows): mask byte [r][g] = query row row0 + r,
// key group (col0 >> 3) + g.  Lane reads its rows r, r + 8 as 64-bit words pre-shifted to its
// column pair: fragment element i is kept iff bit 8 (i >> 2) + (i & 1) of k[(i >> 1) & 1].
__device__ __forceinline__ void draw_qrows(const philox::Drop& d, uint8_t* wm, int b, int h, int row0, int col0,
                                           int lane) {
#pragma unroll
  for (int m = 0; m < 4; ++m)
    wm[lane + 32 * m] = static_cast<uint8_t>(philox::keep8(d, b, h, row0 + (lane >> 3) + 4 * m, (col0 >> 3) + (lane & 7)));
}
__device__ __forceinline__ void read_qrows(const uint8_t* wm, int lane, uint64_t (&k)[2]) {
#pragma unroll
  for (int e = 0; e < 2; ++e)
    k[e] = *reinterpret_cast<const uint64_t*>(wm + 8 * ((lane >> 2) + 8 * e)) >> (2 * (lane & 3));
}
__device__ __forceinline__ bool kept_q(const uint64_t (&k)[2], int i) {
  return (k[(i >> 1) & 1] >> (8 * (i >> 2) + (i & 1))) & 1u;
}
// dK / dV layout (accumulator rows = keys key0 .. key0 + 15 of the warp): mask byte [r][u] = query
// row row0 + r, key group (key0 >> 3) + u.  Lane reads, per 8-query group g, the 4 bytes of its query
// rows 8g + 2 (lane & 3) + {0, 1}, shifted to its key bit: fragment element t is kept iff bit
// 8 (2 (t & 1) + ((t >> 1) & 1)) of k[t >> 2].
__device__ __forceinline__ void draw_keys(const philox::Drop& d, uint8_t* wm, int b, int h, int row0, int key0,
                                          int lane) {
#pragma unroll
  for (int m = 0; m < 4; ++m)
    wm[lane + 32 * m] = static_cast<uint8_t>(philox::keep8(d, b, h, row0 + (lane >> 1) + 16 * m, (key0 >> 3) + (lane & 1)));
}
__device__ __forceinline__ void read_keys(const uint8_t* wm, int lane, uint32_t (&k)[8]) {
#pragma unroll
  for (int g = 0; g < 8; ++g) k[g] = *reinterpret_cast<const uint32_t*>(wm + 16 * g + 4 * (lane & 3)) >> (lane >> 2);
}
__device__ __forceinline__ bool kept_k(const uint32_t (&k)[8], int t) {
  return (k[t >> 2] >> (8 * (2 * (t & 1) + ((t >> 1) & 1)))) & 1u;
}
constexpr int kDropSmem = 1024;              // 128 B per MMA warp, after the barrier block

// --------------------------------------------------------------------------- forward
constexpr int kVFwdSmem = 2 * kVTile + kVStages * 2 * kVTile + 2 * kVTile + 256 + 1024;

// Packed mode: cu_seqlens is device data an earlier kernel may still be writing, so a packed CTA
// reads it after the dependency wait, and leaves before any barrier or TMA if its block starts at
// or past len_b.  -> (len_b, first row of sequence b, live warpgroups of query block qb)
__device__ __forceinline__ bool packed_prologue(const VarP& p, int b, int qb, int& len, int& row_base, int& live) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  len = packed_len(p, b);
  row_base = p.cu[b];
  live = min(2, (len - qb * kVQ + kVB - 1) / kVB);
  return qb * kVQ < len;
}

template <bool kPacked, bool kDrop, bool kCausal>
__device__ __forceinline__ void fwd_var_body(const CUtensorMap& tmQ, const CUtensorMap& tmK,
                                             const CUtensorMap& tmV, const VarArgs<kDrop> p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sQ = smem;                              // warpgroup g: rows 64 g.. of the query block
  uint8_t* ring = smem + 2 * kVTile;               // stage s: K tile, V tile
  uint8_t* sP = ring + kVStages * 2 * kVTile;      // warpgroup g: its [64 x 64] P block
  uint64_t* bar_q = reinterpret_cast<uint64_t*>(sP + 2 * kVTile);
  uint64_t* full = bar_q + 1;
  uint64_t* empty = full + kVStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nqb = (p.S + kVQ - 1) / kVQ;
  const int bh = blockIdx.x / nqb, qb = blockIdx.x % nqb, b = bh / p.H, h = bh % p.H;
  int len = 0, row_base = 0, live;
  if constexpr (kPacked) {
    if (!packed_prologue(p, b, qb, len, row_base, live)) return;
  } else {
    live = live_groups(p.S, qb);
  }
  if (threadIdx.x == 0) {
    ptx::mbar_init(bar_q, 1);
    for (int s = 0; s < kVStages; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], 4 * live);         // every warp of the live warpgroups
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  if constexpr (!kPacked) {
    ptx::pdl_launch_dependents();
    ptx::pdl_wait();
    len = valid_len(p, b);
    row_base = b * p.S;
  }
  const int nkb = key_blocks(len);
  philox::Drop drop{};
  if constexpr (kDrop) drop = drop_of(p);
  if (warp == 8) {
    if (lane == 0) {
      ptx::mbar_expect_tx(bar_q, live * kVTile);
      for (int g = 0; g < live; ++g)
        ptx::tma_load_3d(sQ + g * kVTile, &tmQ, bar_q, h * kD, row_base + qb * kVQ + g * kVB, 0);
      const int nload = kCausal ? min(nkb, 2 * qb + live) : nkb;
      for (int j = 0; j < nload; ++j) {
        const int s = j % kVStages;
        ptx::mbar_wait(&empty[s], ((j / kVStages) & 1) ^ 1);
        uint8_t* st = ring + s * 2 * kVTile;
        ptx::mbar_expect_tx(&full[s], 2 * kVTile);
        ptx::tma_load_3d(st, &tmK, &full[s], h * kD, row_base + j * kVB, 0);
        ptx::tma_load_3d(st + kVTile, &tmV, &full[s], h * kD, row_base + j * kVB, 0);
      }
    }
    return;
  }
  const int g = warp >> 2, w = warp & 3;
  if (g >= live) return;
  const int q0 = qb * kVQ + g * kVB;               // first sequence row of this warpgroup
  const int diag = 2 * qb + g;                     // causal: the last key block this warpgroup reads
  const int nkb_g = kCausal ? min(nkb, diag + 1) : nkb;
  const float sc = p.scale * kLog2e;
  uint8_t* sPg = sP + g * kVTile;
  uint8_t* wmask = reinterpret_cast<uint8_t*>(bar_q) + 256 + 128 * warp;   // kDrop only
  float o[32], m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  wg::zero(o);
  ptx::mbar_wait(bar_q, 0);
#pragma unroll 1
  for (int j = 0; j < nkb_g; ++j) {
    const int s = j % kVStages, kv0 = j * kVB;
    const uint32_t sk = ptx::smem_u32(ring + s * 2 * kVTile);
    ptx::mbar_wait(&full[s], (j / kVStages) & 1);
    float sv[32];
    uint64_t keep[2];
    wg::fence();
    mma_nt64(sv, ptx::smem_u32(sQ + g * kVTile), sk);   // S = Q K^T
    if constexpr (kDrop) {
      wg::commit();
      draw_qrows(drop, wmask, b, h, q0 + 16 * w, kv0, lane);   // while the MMA runs
      wg::wait<0>();
      wg::reg_fence(sv);
      __syncwarp();
      read_qrows(wmask, lane, keep);
    } else {
      run_sync(sv);
    }
    if (kv0 + kVB > len) {                         // the block that straddles len
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (kv0 + wg::frag_col(i, lane) >= len) sv[i] = -INFINITY;
    }
    if (kCausal && j == diag) {                   // key column > query row (same block offset)
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (wg::frag_col(i, lane) > 16 * w + (lane >> 2) + 8 * ((i >> 1) & 1)) sv[i] = -INFINITY;
    }
    // column kv0 < len is valid (causal: key 0 is in block 0), so the new row max is finite and
    // exp2 of (m_old - m_new) is 0 on the first block (m_old = -inf)
    float mx[2] = {m[0], m[1]};
#pragma unroll
    for (int i = 0; i < 32; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], sv[i]);
    float alpha[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      mx[e] = quad_max(mx[e]);
      alpha[e] = exp2f((m[e] - mx[e]) * sc);
      m[e] = mx[e];
      l[e] *= alpha[e];
    }
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int e = (i >> 1) & 1;
      const float p0 = exp2f((sv[i] - m[e]) * sc), p1 = exp2f((sv[i + 1] - m[e]) * sc);
      l[e] += p0 + p1;                             // this thread's columns; quad-summed at the end
      o[i] *= alpha[e];
      o[i + 1] *= alpha[e];
      if constexpr (kDrop)                         // O accumulates the kept P; 1 / (1 - p) at the end
        put2_kmaj(sPg, 16 * w + (lane >> 2) + 8 * e, wg::frag_col(i, lane), kept_q(keep, i) ? p0 : 0.f,
                  kept_q(keep, i + 1) ? p1 : 0.f);
      else
        put2_kmaj(sPg, 16 * w + (lane >> 2) + 8 * e, wg::frag_col(i, lane), p0, p1);
    }
    ptx::fence_proxy_async_smem();                 // P (generic stores) -> wgmma operand reads
    wg_bar(1 + g);
    wg::fence();
    mma_nn64(o, ptx::smem_u32(sPg), sk + kVTile);  // O += P V
    run_sync(o);
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(&empty[s]);
  }
  float inv[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    l[e] = quad_sum(l[e]);
    inv[e] = l[e] > 0.f ? 1.f / l[e] : 0.f;
    if constexpr (kDrop) inv[e] *= drop.scale;
  }
  const long long gbase = static_cast<long long>(row_base) * p.ld + h * kD;
  if constexpr (kPacked)
    store_frag64_rows(o, p.o + gbase, p.ld, q0 + 16 * w, inv[0], inv[1], len);
  else
    store_frag64(o, p.o + gbase, p.ld, q0 + 16 * w, inv[0], inv[1]);
  if ((lane & 3) == 0) {
#pragma unroll
    for (int e = 0; e < 2; ++e)
      p.lse[static_cast<long long>(bh) * p.S + q0 + 16 * w + (lane >> 2) + 8 * e] =
          l[e] > 0.f ? m[e] * p.scale + __logf(l[e]) : 0.f;
  }
}
template <bool kPacked, bool kDrop>
__global__ void __launch_bounds__(kVThreads, 1)
attn_fwd_var_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const VarArgs<kDrop> p) {
  fwd_var_body<kPacked, kDrop, false>(tmQ, tmK, tmV, p);
}
template <bool kDrop>
__global__ void __launch_bounds__(kVThreads, 1)
attn_causal_fwd(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const VarArgs<kDrop> p) {
  fwd_var_body<false, kDrop, true>(tmQ, tmK, tmV, p);
}

// ------------------------------------------------------------------------------- dQ
constexpr int kVDqSmem = 4 * kVTile + kVStages * 2 * kVTile + 2 * kVTile + 256 + 1024;

template <bool kPacked, bool kDrop, bool kCausal>
__device__ __forceinline__ void dq_var_body(const CUtensorMap& tmQ, const CUtensorMap& tmK,
                                            const CUtensorMap& tmV, const CUtensorMap& tmDO,
                                            const VarArgs<kDrop> p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sQ = smem;                              // warpgroup g: Q rows at tile g, dO rows at tile 2 + g
  uint8_t* sDO = smem + 2 * kVTile;
  uint8_t* ring = smem + 4 * kVTile;
  uint8_t* sDS = ring + kVStages * 2 * kVTile;
  uint64_t* bar_q = reinterpret_cast<uint64_t*>(sDS + 2 * kVTile);
  uint64_t* full = bar_q + 1;
  uint64_t* empty = full + kVStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nqb = (p.S + kVQ - 1) / kVQ;
  const int bh = blockIdx.x / nqb, qb = blockIdx.x % nqb, b = bh / p.H, h = bh % p.H;
  int len = 0, row_base = 0, live;
  if constexpr (kPacked) {
    if (!packed_prologue(p, b, qb, len, row_base, live)) return;
  } else {
    live = live_groups(p.S, qb);
  }
  if (threadIdx.x == 0) {
    ptx::mbar_init(bar_q, 1);
    for (int s = 0; s < kVStages; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], 4 * live);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  if constexpr (!kPacked) {
    ptx::pdl_launch_dependents();
    ptx::pdl_wait();
    len = valid_len(p, b);
    row_base = b * p.S;
  }
  const int nkb = key_blocks(len);
  philox::Drop drop{};
  if constexpr (kDrop) drop = drop_of(p);
  if (warp == 8) {
    if (lane == 0) {
      ptx::mbar_expect_tx(bar_q, 2 * live * kVTile);
      for (int g = 0; g < live; ++g) {
        ptx::tma_load_3d(sQ + g * kVTile, &tmQ, bar_q, h * kD, row_base + qb * kVQ + g * kVB, 0);
        ptx::tma_load_3d(sDO + g * kVTile, &tmDO, bar_q, h * kD, row_base + qb * kVQ + g * kVB, 0);
      }
      const int nload = kCausal ? min(nkb, 2 * qb + live) : nkb;   // as in the forward
      for (int j = 0; j < nload; ++j) {
        const int s = j % kVStages;
        ptx::mbar_wait(&empty[s], ((j / kVStages) & 1) ^ 1);
        uint8_t* st = ring + s * 2 * kVTile;
        ptx::mbar_expect_tx(&full[s], 2 * kVTile);
        ptx::tma_load_3d(st, &tmK, &full[s], h * kD, row_base + j * kVB, 0);
        ptx::tma_load_3d(st + kVTile, &tmV, &full[s], h * kD, row_base + j * kVB, 0);
      }
    }
    return;
  }
  const int g = warp >> 2, w = warp & 3;
  if (g >= live) return;
  const int q0 = qb * kVQ + g * kVB;
  const int diag = 2 * qb + g;
  const int nkb_g = kCausal ? min(nkb, diag + 1) : nkb;
  const float sc = p.scale * kLog2e;
  uint8_t* sDSg = sDS + g * kVTile;
  uint8_t* wmask = reinterpret_cast<uint8_t*>(bar_q) + 256 + 128 * warp;   // kDrop only
  // delta = rowsum(dO * O) of rows r0, r0 + 8: each lane of a quad sums 16 of the 64 columns
  float delta[2], lse2[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int r = q0 + 16 * w + (lane >> 2) + 8 * e;
    const long long goff = (static_cast<long long>(row_base) + r) * p.ld + h * kD + 16 * (lane & 3);
    const uint4* o4 = reinterpret_cast<const uint4*>(p.o_in + goff);
    const uint4* d4 = reinterpret_cast<const uint4*>(p.dout_g + goff);
    float acc = 0.f;
    if (!kPacked || r < len) {                     // packed: rows past len_b are another sequence's, or past T
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const uint4 a = o4[j], c = d4[j];
        const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, cw[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 fa = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&aw[t]));
          const float2 fc = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&cw[t]));
          acc += fa.x * fc.x + fa.y * fc.y;
        }
      }
    }
    delta[e] = quad_sum(acc);
    const long long li = static_cast<long long>(bh) * p.S + r;
    lse2[e] = p.lse[li] * kLog2e;
    if ((lane & 3) == 0) p.delta[li] = delta[e];
  }
  float acc[32];
  wg::zero(acc);
  ptx::mbar_wait(bar_q, 0);
#pragma unroll 1
  for (int j = 0; j < nkb_g; ++j) {
    const int s = j % kVStages, kv0 = j * kVB;
    const uint32_t sk = ptx::smem_u32(ring + s * 2 * kVTile);
    const bool on_diag = kCausal && j == diag;
    ptx::mbar_wait(&full[s], (j / kVStages) & 1);
    float sv[32], dp[32];
    uint64_t keep[2];
    wg::fence();
    mma_nt64(sv, ptx::smem_u32(sQ + g * kVTile), sk);             // S  = Q K^T
    mma_nt64(dp, ptx::smem_u32(sDO + g * kVTile), sk + kVTile);   // dP = dO V^T
    if constexpr (kDrop) {
      wg::commit();
      draw_qrows(drop, wmask, b, h, q0 + 16 * w, kv0, lane);   // while the MMAs run
      wg::wait<0>();
      wg::reg_fence(sv);
      wg::reg_fence(dp);
      __syncwarp();
      read_qrows(wmask, lane, keep);
    } else {
      run_sync2(sv, dp);
    }
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int e = (i >> 1) & 1, col = wg::frag_col(i, lane), r = 16 * w + (lane >> 2) + 8 * e;
      const bool v0 = kv0 + col < len && !(on_diag && col > r), v1 = kv0 + col + 1 < len && !(on_diag && col + 1 > r);
      const float p0 = v0 ? exp2f(sv[i] * sc - lse2[e]) : 0.f;
      const float p1 = v1 ? exp2f(sv[i + 1] * sc - lse2[e]) : 0.f;
      float g0 = dp[i], g1 = dp[i + 1];            // dropout: dS = P (Z dP - delta)
      if constexpr (kDrop) {
        g0 = kept_q(keep, i) ? g0 * drop.scale : 0.f;
        g1 = kept_q(keep, i + 1) ? g1 * drop.scale : 0.f;
      }
      const float d0 = v0 ? p0 * (g0 - delta[e]) * p.scale : 0.f;
      const float d1 = v1 ? p1 * (g1 - delta[e]) * p.scale : 0.f;
      put2_kmaj(sDSg, 16 * w + (lane >> 2) + 8 * e, col, d0, d1);
    }
    ptx::fence_proxy_async_smem();
    wg_bar(1 + g);
    wg::fence();
    mma_nn64(acc, ptx::smem_u32(sDSg), sk);        // dQ += dS K
    run_sync(acc);
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(&empty[s]);
  }
  __nv_bfloat16* dq = p.dq + static_cast<long long>(row_base) * p.ld + h * kD;
  if constexpr (kPacked)
    store_frag64_rows(acc, dq, p.ld, q0 + 16 * w, 1.f, 1.f, len);
  else
    store_frag64(acc, dq, p.ld, q0 + 16 * w, 1.f, 1.f);
}
template <bool kPacked, bool kDrop>
__global__ void __launch_bounds__(kVThreads, 1)
attn_dq_var_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                   const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                   const VarArgs<kDrop> p) {
  dq_var_body<kPacked, kDrop, false>(tmQ, tmK, tmV, tmDO, p);
}
template <bool kDrop>
__global__ void __launch_bounds__(kVThreads, 1)
attn_causal_dq(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
               const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
               const VarArgs<kDrop> p) {
  dq_var_body<false, kDrop, true>(tmQ, tmK, tmV, tmDO, p);
}

// ---------------------------------------------------------------------------- dK / dV
constexpr int kVStageKV = 2 * kVTile + 1024;       // Q tile, dO tile, 64 lse + 64 delta (1 KB-aligned)
constexpr int kVKvSmem = 2 * kVTile + kVStages * kVStageKV + 2 * kVTile + 256 + 1024;

template <bool kPacked, bool kDrop, bool kCausal>
__device__ __forceinline__ void dkv_var_body(const CUtensorMap& tmQ, const CUtensorMap& tmK,
                                             const CUtensorMap& tmV, const CUtensorMap& tmDO,
                                             const VarArgs<kDrop> p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sK = smem;
  uint8_t* sV = smem + kVTile;
  uint8_t* ring = smem + 2 * kVTile;
  uint8_t* sPt = ring + kVStages * kVStageKV;      // P^T block (keys x queries), K-major
  uint8_t* sDSt = sPt + kVTile;                    // dS^T block
  uint64_t* bar_k = reinterpret_cast<uint64_t*>(sDSt + kVTile);
  uint64_t* full = bar_k + 1;
  uint64_t* empty = full + kVStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nb = p.S / kVB;
  const int bh = blockIdx.x / nb, kb = blockIdx.x % nb, b = bh / p.H, h = bh % p.H;
  const int kv0 = kb * kVB;
  int len = 0, row_base = 0;
  if constexpr (kPacked) {                         // see packed_prologue
    ptx::pdl_launch_dependents();
    ptx::pdl_wait();
    len = packed_len(p, b);
    row_base = p.cu[b];
    if (kv0 >= len) return;
  }
  if (threadIdx.x == 0) {
    ptx::mbar_init(bar_k, 1);
    for (int s = 0; s < kVStages; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], 4);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  if constexpr (!kPacked) {
    ptx::pdl_launch_dependents();
    ptx::pdl_wait();
    len = valid_len(p, b);
    row_base = b * p.S;
  }
  const long long gbase = static_cast<long long>(row_base) * p.ld + h * kD;
  if (!kPacked && kv0 >= len) {                    // every key of the block is masked
    for (int idx = threadIdx.x; idx < kVB * 8; idx += kVThreadsKV) {
      const long long off = gbase + (kv0 + (idx >> 3)) * p.ld + (idx & 7) * 8;
      *reinterpret_cast<uint4*>(p.dk + off) = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(p.dv + off) = make_uint4(0, 0, 0, 0);
    }
    return;
  }
  // query blocks: padded mode computes every one (padded query rows carry gradient, as in SDPA),
  // packed mode only those holding rows of the sequence
  const int nqb = kPacked ? key_blocks(len) : nb;
  const int qb0 = kCausal ? kb : 0;               // causal: query blocks below kb see none of these keys
  const long long lrow = static_cast<long long>(bh) * p.S;
  philox::Drop drop{};
  if constexpr (kDrop) drop = drop_of(p);
  if (warp == 4) {
    if (lane == 0) {
      ptx::mbar_expect_tx(bar_k, 2 * kVTile);
      ptx::tma_load_3d(sK, &tmK, bar_k, h * kD, row_base + kv0, 0);
      ptx::tma_load_3d(sV, &tmV, bar_k, h * kD, row_base + kv0, 0);
      for (int i = qb0; i < nqb; ++i) {
        const int n = i - qb0, s = n % kVStages;
        ptx::mbar_wait(&empty[s], ((n / kVStages) & 1) ^ 1);
        uint8_t* st = ring + s * kVStageKV;
        ptx::mbar_expect_tx(&full[s], 2 * kVTile + 2 * kVB * 4);
        ptx::tma_load_3d(st, &tmQ, &full[s], h * kD, row_base + i * kVB, 0);
        ptx::tma_load_3d(st + kVTile, &tmDO, &full[s], h * kD, row_base + i * kVB, 0);
        ptx::bulk_load(st + 2 * kVTile, p.lse + lrow + i * kVB, kVB * 4, &full[s]);
        ptx::bulk_load(st + 2 * kVTile + kVB * 4, p.delta + lrow + i * kVB, kVB * 4, &full[s]);
      }
    }
    return;
  }
  const int w = warp;
  const float sc = p.scale * kLog2e;
  const int m0 = 16 * w + (lane >> 2);             // this thread's key rows m0, m0 + 8 of the block
  const bool valid[2] = {kv0 + m0 < len, kv0 + m0 + 8 < len};
  uint8_t* wmask = reinterpret_cast<uint8_t*>(bar_k) + 256 + 128 * warp;   // kDrop only
  float dk[32], dv[32];
  wg::zero(dk);
  wg::zero(dv);
  ptx::mbar_wait(bar_k, 0);
#pragma unroll 1
  for (int i = qb0; i < nqb; ++i) {
    const int n = i - qb0, s = n % kVStages;
    uint8_t* st = ring + s * kVStageKV;
    const uint32_t sq = ptx::smem_u32(st), sdo = sq + kVTile;
    const bool on_diag = kCausal && i == kb;
    ptx::mbar_wait(&full[s], (n / kVStages) & 1);
    float sv[32], dp[32];
    uint32_t keep[8];
    wg::fence();
    mma_nt64(sv, ptx::smem_u32(sK), sq);           // S^T  = K Q^T
    mma_nt64(dp, ptx::smem_u32(sV), sdo);          // dP^T = V dO^T
    if constexpr (kDrop) {
      wg::commit();
      draw_keys(drop, wmask, b, h, i * kVB, kv0 + 16 * w, lane);   // while the MMAs run
      wg::wait<0>();
      wg::reg_fence(sv);
      wg::reg_fence(dp);
      __syncwarp();
      read_keys(wmask, lane, keep);
    } else {
      run_sync2(sv, dp);
    }
    const float* s_lse = reinterpret_cast<const float*>(st + 2 * kVTile);
    const float* s_delta = s_lse + kVB;
#pragma unroll
    for (int t = 0; t < 32; t += 2) {
      const int e = (t >> 1) & 1, col = wg::frag_col(t, lane);   // col: query row of the block
      const float2 L = *reinterpret_cast<const float2*>(s_lse + col);
      const float2 Dl = *reinterpret_cast<const float2*>(s_delta + col);
      bool v0 = valid[e] && !(on_diag && col < m0 + 8 * e), v1 = valid[e] && !(on_diag && col + 1 < m0 + 8 * e);
      if constexpr (kPacked) {                     // query rows past len_b: another sequence, or past T
        v0 = v0 && i * kVB + col < len;
        v1 = v1 && i * kVB + col + 1 < len;
      }
      const float p0 = v0 ? exp2f(sv[t] * sc - L.x * kLog2e) : 0.f;
      const float p1 = v1 ? exp2f(sv[t + 1] * sc - L.y * kLog2e) : 0.f;
      float g0 = dp[t], g1 = dp[t + 1], z0 = p0, z1 = p1;   // dropout: dV += (P Z)^T dO (1 / (1 - p) at
      if constexpr (kDrop) {                                //   the store), dS = P (Z dP - delta)
        const bool k0 = kept_k(keep, t), k1 = kept_k(keep, t + 1);
        g0 = k0 ? g0 * drop.scale : 0.f;
        g1 = k1 ? g1 * drop.scale : 0.f;
        z0 = k0 ? p0 : 0.f;
        z1 = k1 ? p1 : 0.f;
      }
      const float d0 = v0 ? p0 * (g0 - Dl.x) * p.scale : 0.f;
      const float d1 = v1 ? p1 * (g1 - Dl.y) * p.scale : 0.f;
      put2_kmaj(sPt, m0 + 8 * e, col, z0, z1);
      put2_kmaj(sDSt, m0 + 8 * e, col, d0, d1);
    }
    ptx::fence_proxy_async_smem();
    wg_bar(1);
    wg::fence();
    mma_nn64(dv, ptx::smem_u32(sPt), sdo);         // dV += P^T dO
    mma_nn64(dk, ptx::smem_u32(sDSt), sq);         // dK += dS^T Q
    run_sync2(dv, dk);
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(&empty[s]);
  }
  if constexpr (kDrop) {                           // dV = (P Z)^T dO: the 1 / (1 - p) of Z
#pragma unroll
    for (int t = 0; t < 32; ++t) dv[t] *= drop.scale;
  }
  if constexpr (kPacked) {
    store_frag64_rows(dk, p.dk + gbase, p.ld, kv0 + 16 * w, 1.f, 1.f, len);
    store_frag64_rows(dv, p.dv + gbase, p.ld, kv0 + 16 * w, 1.f, 1.f, len);
  } else {
    store_frag64(dk, p.dk + gbase, p.ld, kv0 + 16 * w, 1.f, 1.f);
    store_frag64(dv, p.dv + gbase, p.ld, kv0 + 16 * w, 1.f, 1.f);
  }
}
template <bool kPacked, bool kDrop>
__global__ void __launch_bounds__(kVThreadsKV, 1)
attn_dkv_var_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                    const VarArgs<kDrop> p) {
  dkv_var_body<kPacked, kDrop, false>(tmQ, tmK, tmV, tmDO, p);
}
template <bool kDrop>
__global__ void __launch_bounds__(kVThreadsKV, 1)
attn_causal_dkv(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                const VarArgs<kDrop> p) {
  dkv_var_body<false, kDrop, true>(tmQ, tmK, tmV, tmDO, p);
}

cudaError_t head_map(CUtensorMap* out, const void* ptr, long long ld, long long rows, int hd, int box_rows) {
  GemmOperand op{ptr, ld, 0, false};
  return gemm_make_operand_map(out, op, DType::BF16, static_cast<int>(rows), hd, 1, box_rows);
}

bool var_shape(int S, int D) { return D == kD && S % kVB == 0 && S >= kVB && S <= kVMaxS; }

template <typename K>
cudaError_t set_smem_once(K kernel, int bytes, bool& done) {
  if (done) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  done = e == cudaSuccess;
  return e;
}

// -> 1: dropout on (fields of vp set), 0: off, -1: invalid arguments
int set_dropout(VarPDrop& vp, const DropoutArgs* drop) {
  if (drop == nullptr || drop->p == 0.f) return 0;
  if (!(drop->p > 0.f && drop->p < 1.f) || drop->step == nullptr || drop->site >= (1u << 24)) return -1;
  vp.drop_step = drop->step;
  vp.drop_add = drop->step_add;
  vp.seed_lo = static_cast<uint32_t>(drop->seed);
  vp.seed_hi = static_cast<uint32_t>(drop->seed >> 32);
  vp.site = drop->site;
  vp.thr = philox::threshold(drop->p);
  vp.dscale = 1.f / (1.f - drop->p);
  return 1;
}

template <bool kPacked, bool kDrop, bool kCausal = false>
cudaError_t launch_fwd_var(int grid, cudaStream_t stream, const CUtensorMap& tq, const CUtensorMap& tk,
                           const CUtensorMap& tv, const VarArgs<kDrop>& vp) {
  static bool cfg = false;
  constexpr int smem = kVFwdSmem + (kDrop ? kDropSmem : 0);
  constexpr auto kernel = kCausal ? attn_causal_fwd<kDrop> : attn_fwd_var_kernel<kPacked, kDrop>;
  cudaError_t e;
  if ((e = set_smem_once(kernel, smem, cfg)) != cudaSuccess) return e;
  note_launch();
  return launch_pdl(kernel, dim3(grid), dim3(kVThreads), smem, stream, tq, tk, tv, vp);
}

// dQ (and delta) over grid_q CTAs, then dK / dV over grid_kv CTAs
template <bool kPacked, bool kDrop, bool kCausal = false>
cudaError_t launch_bwd_var(int grid_q, int grid_kv, cudaStream_t stream, const CUtensorMap& tq, const CUtensorMap& tk,
                           const CUtensorMap& tv, const CUtensorMap& tdo, const VarArgs<kDrop>& vp) {
  static bool dq_cfg = false, kv_cfg = false;
  constexpr int smem_q = kVDqSmem + (kDrop ? kDropSmem : 0), smem_kv = kVKvSmem + (kDrop ? kDropSmem : 0);
  constexpr auto kq = kCausal ? attn_causal_dq<kDrop> : attn_dq_var_kernel<kPacked, kDrop>;
  constexpr auto kkv = kCausal ? attn_causal_dkv<kDrop> : attn_dkv_var_kernel<kPacked, kDrop>;
  cudaError_t e;
  if ((e = set_smem_once(kq, smem_q, dq_cfg)) != cudaSuccess) return e;
  if ((e = set_smem_once(kkv, smem_kv, kv_cfg)) != cudaSuccess) return e;
  note_launch();
  e = launch_pdl(kq, dim3(grid_q), dim3(kVThreads), smem_q, stream, tq, tk, tv, tdo, vp);
  if (e != cudaSuccess) return e;
  note_launch();   // reads the delta rows the dQ kernel wrote
  return launch_pdl(kkv, dim3(grid_kv), dim3(kVThreadsKV), smem_kv, stream, tq, tk, tv, tdo, vp);
}

}  // namespace

cudaError_t attention_fwd_sm100(const void* q, const void* k, const void* v, void* o, float* lse, int B, int S,
                                int H, int D, long long ld, float scale, cudaStream_t stream,
                                const int32_t* lengths, const DropoutArgs* drop, bool causal) {
  bind_context_once();
  if (ld % 8 != 0 || B <= 0 || H <= 0 || (causal && lengths != nullptr)) return cudaErrorNotSupported;
  VarPDrop vp{};
  const int dropping = set_dropout(vp, drop);
  if (dropping < 0) return cudaErrorInvalidValue;
  // the one-CTA-per-head kernel (no dropout or causal mask there: unmasked S = 128 with either runs
  // the tiled kernels)
  const bool whole = lengths == nullptr && S == kS && D == kD && !dropping && !causal;
  if (!whole && !var_shape(S, D)) return cudaErrorNotSupported;
  CUtensorMap tq, tk, tv;
  cudaError_t e;
  const long long rows = static_cast<long long>(B) * S;
  const int box = whole ? kS : kVB;
  if ((e = head_map(&tq, q, ld, rows, H * D, box)) != cudaSuccess) return e;
  if ((e = head_map(&tk, k, ld, rows, H * D, box)) != cudaSuccess) return e;
  if ((e = head_map(&tv, v, ld, rows, H * D, box)) != cudaSuccess) return e;
  if (!whole) {
    vp.S = S; vp.H = H; vp.ld = ld; vp.scale = scale; vp.lengths = lengths;
    vp.o = static_cast<__nv_bfloat16*>(o); vp.lse = lse;
    const int grid = B * H * ((S + kVQ - 1) / kVQ);
    const VarP& np = vp;
    if (causal)
      return dropping ? launch_fwd_var<false, true, true>(grid, stream, tq, tk, tv, vp)
                      : launch_fwd_var<false, false, true>(grid, stream, tq, tk, tv, np);
    return dropping ? launch_fwd_var<false, true>(grid, stream, tq, tk, tv, vp)
                    : launch_fwd_var<false, false>(grid, stream, tq, tk, tv, np);
  }
  AttnP p{};
  p.H = H; p.ld = ld; p.scale = scale; p.o = static_cast<__nv_bfloat16*>(o); p.lse = lse;
  static bool cfg = false;
  if (!cfg) {
    e = cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFwdSmem);
    if (e != cudaSuccess) return e;
    cfg = true;
  }
  note_launch();
  return launch_pdl(attn_fwd_kernel, dim3(B * H), dim3(kThreads), kFwdSmem, stream, tq, tk, tv, p);
}

cudaError_t attention_bwd_sm100(const void* q, const void* k, const void* v, const void* o, const void* dout,
                                const float* lse, void* dq, void* dk, void* dv, int B, int S, int H, int D,
                                long long ld, float scale, cudaStream_t stream, float* delta,
                                const int32_t* lengths, const DropoutArgs* drop, bool causal) {
  bind_context_once();
  if (ld % 8 != 0 || B <= 0 || H <= 0 || (causal && lengths != nullptr)) return cudaErrorNotSupported;
  VarPDrop vp{};
  const int dropping = set_dropout(vp, drop);
  if (dropping < 0) return cudaErrorInvalidValue;
  const bool whole = lengths == nullptr && S == kS && D == kD && !dropping && !causal;
  if (!whole && !var_shape(S, D)) return cudaErrorNotSupported;
  if (!whole && delta == nullptr) return cudaErrorInvalidValue;
  CUtensorMap tq, tk, tv, tdo;
  cudaError_t e;
  const long long rows = static_cast<long long>(B) * S;
  const int box = whole ? kS : kVB;
  if ((e = head_map(&tq, q, ld, rows, H * D, box)) != cudaSuccess) return e;
  if ((e = head_map(&tk, k, ld, rows, H * D, box)) != cudaSuccess) return e;
  if ((e = head_map(&tv, v, ld, rows, H * D, box)) != cudaSuccess) return e;
  if ((e = head_map(&tdo, dout, ld, rows, H * D, box)) != cudaSuccess) return e;
  if (!whole) {
    vp.S = S; vp.H = H; vp.ld = ld; vp.scale = scale; vp.lengths = lengths;
    vp.lse = const_cast<float*>(lse); vp.delta = delta;
    vp.o_in = static_cast<const __nv_bfloat16*>(o); vp.dout_g = static_cast<const __nv_bfloat16*>(dout);
    vp.dq = static_cast<__nv_bfloat16*>(dq); vp.dk = static_cast<__nv_bfloat16*>(dk);
    vp.dv = static_cast<__nv_bfloat16*>(dv);
    const int gq = B * H * ((S + kVQ - 1) / kVQ), gkv = B * H * (S / kVB);
    const VarP& np = vp;
    if (causal)
      return dropping ? launch_bwd_var<false, true, true>(gq, gkv, stream, tq, tk, tv, tdo, vp)
                      : launch_bwd_var<false, false, true>(gq, gkv, stream, tq, tk, tv, tdo, np);
    return dropping ? launch_bwd_var<false, true>(gq, gkv, stream, tq, tk, tv, tdo, vp)
                    : launch_bwd_var<false, false>(gq, gkv, stream, tq, tk, tv, tdo, np);
  }
  AttnP p{};
  p.H = H; p.ld = ld; p.scale = scale; p.lse = const_cast<float*>(lse);
  p.o_in = static_cast<const __nv_bfloat16*>(o); p.dout_g = static_cast<const __nv_bfloat16*>(dout);
  p.dq = static_cast<__nv_bfloat16*>(dq); p.dk = static_cast<__nv_bfloat16*>(dk); p.dv = static_cast<__nv_bfloat16*>(dv);
  static bool cfg = false;
  if (!cfg) {
    e = cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kBwdSmem);
    if (e != cudaSuccess) return e;
    cfg = true;
  }
  note_launch();
  return launch_pdl(attn_bwd_kernel, dim3(B * H), dim3(kThreads), kBwdSmem, stream, tq, tk, tv, tdo, p);
}

namespace {
bool packed_shape(int B, int T, int max_seqlen, int H, int D, long long ld) {
  return D == kD && ld % 8 == 0 && B > 0 && T > 0 && H > 0 && max_seqlen >= 1 && max_seqlen <= kVMaxS;
}
VarP packed_params(const int32_t* cu_seqlens, int T, int max_seqlen, int H, long long ld, float scale) {
  VarP vp{};
  vp.S = (max_seqlen + kVB - 1) / kVB * kVB;
  vp.H = H; vp.ld = ld; vp.scale = scale; vp.cu = cu_seqlens; vp.T = T;
  return vp;
}
}  // namespace

cudaError_t attention_packed_fwd_sm100(const void* q, const void* k, const void* v, void* o, float* lse,
                                       const int32_t* cu_seqlens, int B, int T, int max_seqlen, int H, int D,
                                       long long ld, float scale, cudaStream_t stream, const DropoutArgs* drop) {
  bind_context_once();
  if (!packed_shape(B, T, max_seqlen, H, D, ld)) return cudaErrorNotSupported;
  if (cu_seqlens == nullptr) return cudaErrorInvalidValue;
  CUtensorMap tq, tk, tv;
  cudaError_t e;
  if ((e = head_map(&tq, q, ld, T, H * D, kVB)) != cudaSuccess) return e;
  if ((e = head_map(&tk, k, ld, T, H * D, kVB)) != cudaSuccess) return e;
  if ((e = head_map(&tv, v, ld, T, H * D, kVB)) != cudaSuccess) return e;
  VarPDrop vp{};
  static_cast<VarP&>(vp) = packed_params(cu_seqlens, T, max_seqlen, H, ld, scale);
  const int dropping = set_dropout(vp, drop);
  if (dropping < 0) return cudaErrorInvalidValue;
  vp.o = static_cast<__nv_bfloat16*>(o); vp.lse = lse;
  const int grid = B * H * ((vp.S + kVQ - 1) / kVQ);
  return dropping ? launch_fwd_var<true, true>(grid, stream, tq, tk, tv, vp)
                  : launch_fwd_var<true, false>(grid, stream, tq, tk, tv, static_cast<const VarP&>(vp));
}

cudaError_t attention_packed_bwd_sm100(const void* q, const void* k, const void* v, const void* o, const void* dout,
                                       const float* lse, void* dq, void* dk, void* dv, const int32_t* cu_seqlens,
                                       int B, int T, int max_seqlen, int H, int D, long long ld, float scale,
                                       cudaStream_t stream, float* delta, const DropoutArgs* drop) {
  bind_context_once();
  if (!packed_shape(B, T, max_seqlen, H, D, ld)) return cudaErrorNotSupported;
  if (cu_seqlens == nullptr || delta == nullptr) return cudaErrorInvalidValue;
  CUtensorMap tq, tk, tv, tdo;
  cudaError_t e;
  if ((e = head_map(&tq, q, ld, T, H * D, kVB)) != cudaSuccess) return e;
  if ((e = head_map(&tk, k, ld, T, H * D, kVB)) != cudaSuccess) return e;
  if ((e = head_map(&tv, v, ld, T, H * D, kVB)) != cudaSuccess) return e;
  if ((e = head_map(&tdo, dout, ld, T, H * D, kVB)) != cudaSuccess) return e;
  VarPDrop vp{};
  static_cast<VarP&>(vp) = packed_params(cu_seqlens, T, max_seqlen, H, ld, scale);
  const int dropping = set_dropout(vp, drop);
  if (dropping < 0) return cudaErrorInvalidValue;
  vp.lse = const_cast<float*>(lse); vp.delta = delta;
  vp.o_in = static_cast<const __nv_bfloat16*>(o); vp.dout_g = static_cast<const __nv_bfloat16*>(dout);
  vp.dq = static_cast<__nv_bfloat16*>(dq); vp.dk = static_cast<__nv_bfloat16*>(dk);
  vp.dv = static_cast<__nv_bfloat16*>(dv);
  const int gq = B * H * ((vp.S + kVQ - 1) / kVQ), gkv = B * H * (vp.S / kVB);
  return dropping ? launch_bwd_var<true, true>(gq, gkv, stream, tq, tk, tv, tdo, vp)
                  : launch_bwd_var<true, false>(gq, gkv, stream, tq, tk, tv, tdo, static_cast<const VarP&>(vp));
}

}  // namespace bflc
