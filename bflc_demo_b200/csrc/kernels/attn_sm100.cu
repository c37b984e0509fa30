// Fused multi-head self-attention for seq_len = 128, head_dim = 64 (BERT-base, BASELINE.json
// config #5): one CTA per (batch, head) = one warpgroup, every GEMM a Hopper wgmma with register
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

#include "bflc_kernels.h"
#include "epi_common.cuh"
#include "launch.cuh"
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

cudaError_t head_map(CUtensorMap* out, const void* ptr, long long ld, long long rows, int hd) {
  GemmOperand op{ptr, ld, 0, false};
  return gemm_make_operand_map(out, op, DType::BF16, static_cast<int>(rows), hd, 1, kS);
}

}  // namespace

cudaError_t attention_fwd_sm100(const void* q, const void* k, const void* v, void* o, float* lse, int B, int S,
                                int H, int D, long long ld, float scale, cudaStream_t stream) {
  bind_context_once();
  if (S != kS || D != kD || ld % 8 != 0 || B <= 0 || H <= 0) return cudaErrorNotSupported;
  CUtensorMap tq, tk, tv;
  cudaError_t e;
  const long long rows = static_cast<long long>(B) * S;
  if ((e = head_map(&tq, q, ld, rows, H * D)) != cudaSuccess) return e;
  if ((e = head_map(&tk, k, ld, rows, H * D)) != cudaSuccess) return e;
  if ((e = head_map(&tv, v, ld, rows, H * D)) != cudaSuccess) return e;
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
                                long long ld, float scale, cudaStream_t stream) {
  bind_context_once();
  if (S != kS || D != kD || ld % 8 != 0 || B <= 0 || H <= 0) return cudaErrorNotSupported;
  CUtensorMap tq, tk, tv, tdo;
  cudaError_t e;
  const long long rows = static_cast<long long>(B) * S;
  if ((e = head_map(&tq, q, ld, rows, H * D)) != cudaSuccess) return e;
  if ((e = head_map(&tk, k, ld, rows, H * D)) != cudaSuccess) return e;
  if ((e = head_map(&tv, v, ld, rows, H * D)) != cudaSuccess) return e;
  if ((e = head_map(&tdo, dout, ld, rows, H * D)) != cudaSuccess) return e;
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

}  // namespace bflc
