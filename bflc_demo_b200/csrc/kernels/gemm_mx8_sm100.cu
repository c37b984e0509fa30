// Block-scaled fp8 GEMM (OCP MXFP8: e4m3 elements, one UE8M0 scale per 32 K-elements) on
// Hopper wgmma:  D (M x N) = alpha * (A .* SFA) (B .* SFB)^T [+ bias] [act]
//
// A [M, K] and B [N, K] are K-major e4m3, staged by TMA into 128-byte-swizzled smem (one
// K-block = 128 elements = one swizzle row).  The quantiser (k_quantize_mx8 below) writes the
// scale factors in a chunked layout -- per (128-row block, 128-K block) a 512-byte chunk whose
// byte [r%32][r/32][k/32] is the scale of row r, K-group k -- and a `cp.async.bulk` drops the
// chunks into smem with the same mbarrier transaction as the operand tiles.  Hopper has no
// block-scaled MMA: the MMA warpgroup widens each landed stage to f16 (exact, wg::widen_e4m3_tile;
// the f16 wgmma accumulates in full fp32, the e4m3 one does not), then every K-group of 32 is two
// m64n64k16 wgmma into a scratch fragment, added to the fp32 accumulator with the product of its
// row's and its column's scale (wg::mx_accumulate) -- the same sum the block-scaled instruction
// forms.
//
//   warps 0-3  MMA warpgroup (128 x 64 tile = two m64 halves)   warp 4  producer (TMA + bulk SF)
//   warps 5-8  epilogue (accumulator tile -> bias/act -> smem staging -> coalesced stores)
//
// Reference parity: the reference trains in fp32 on CPU (python-sdk/main.py:120-123); BASELINE.json
// names block-scaled fp8 for the MLP / LeNet-5 configs, this is that compute path.
#include <cuda_bf16.h>
#include <cuda_fp8.h>

#include <cstring>

#include "bflc_kernels.h"
#include "epi_common.cuh"
#include "launch.cuh"
#include "sm100_ptx.cuh"
#include "wgmma.cuh"

namespace bflc {

namespace {

constexpr int kBM = 128;
constexpr int kBK = 128;                 // fp8 elements per K-block (= 128 bytes)
using epi::kSfChunk;                     // bytes of scale factors per (128 rows, 128 K)
using epi::kStgLd;
using epi::kStgBytes;
constexpr int kBarBytes = 256;
constexpr int kThreads = 288;
constexpr int kProducerWarp = 4, kEpiWarp0 = 5;

template <int BN> struct Cfg {
  static constexpr int kStages = 3;
  static constexpr int kABytes = kBM * 128, kBBytes = BN * 128;
  static constexpr int kTileStage = kABytes + kBBytes;
  static constexpr int kSfbBytes = kSfChunk;   // the tile's B rows lie in one 128-row chunk
  static constexpr int kSfStage = kSfChunk + kSfbBytes;
  static constexpr int kTiles = kStages * kTileStage;
  static constexpr int kSfOff = kTiles;
  static constexpr int kBarOff = kSfOff + kStages * kSfStage;
  static constexpr int kStgOff = kBarOff + kBarBytes;
  static constexpr int kBiasOff = kStgOff + kStgBytes;
  static constexpr int kAccPitch = BN + 4;
  static constexpr int kAccOff = kBiasOff + BN * 4;
  // f16 copies of A (32 KB) and B; 1024-aligned like every 128B-swizzled operand tile
  static constexpr int kWideOff = (kAccOff + kBM * kAccPitch * 4 + 1023) / 1024 * 1024;
  static constexpr int kWideA = kBM * 256, kWideB = BN * 256;
  static constexpr int kSmem = kWideOff + kWideA + kWideB + 1024;
  static constexpr uint32_t kTxBytes = kTileStage + kSfStage;
  static_assert(kSmem <= 227 * 1024, "shared memory budget");
};

struct PM {
  int M, N, K, k_blocks;
  const uint8_t* sfa; const uint8_t* sfb;   // canonical chunk arrays [row_block][k_block][512]
  void* d; int d_dtype; long long ldd; float alpha;
  const float* bias; int act;
};

using epi::bulk_g2s;
__device__ __forceinline__ uint32_t pack2(float a, float b) { return epi::pack_bf16x2(a, b); }
__device__ __forceinline__ float gelu_f(float x) {
  return 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
}

template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_mx8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const PM p) {
  using C = Cfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::kBarOff);
  uint64_t* empty_bar = full_bar + C::kStages;
  uint64_t* accum_bar = empty_bar + C::kStages;
  float* stage_base = reinterpret_cast<float*>(smem + C::kStgOff);
  float* sbias = reinterpret_cast<float*>(smem + C::kBiasOff);
  const wg::AccTile at{reinterpret_cast<float*>(smem + C::kAccOff), C::kAccPitch};

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * BN;
  ptx::pdl_launch_dependents();

  if (warp == 0 && lane == 0) {
    ptx::tma_prefetch_desc(&tmA);
    ptx::tma_prefetch_desc(&tmB);
    for (int s = 0; s < C::kStages; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 128);
    }
    ptx::mbar_init(accum_bar, 128);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  const int n_kb = p.k_blocks;
  ptx::pdl_wait();

  if (warp == kProducerWarp) {
    const uint8_t* sfa_src = p.sfa + static_cast<long long>(blockIdx.x) * n_kb * kSfChunk;
    const uint8_t* sfb_src = p.sfb + static_cast<long long>(n0 >> 7) * n_kb * kSfChunk;
    for (int i = 0; i < n_kb; ++i) {
      const int s = i % C::kStages;
      const uint32_t ph = (i / C::kStages) & 1;
      ptx::mbar_wait(&empty_bar[s], ph ^ 1);
      if (ptx::elect_one()) {
        uint8_t* sa = smem + s * C::kTileStage;
        uint8_t* sf = smem + C::kSfOff + s * C::kSfStage;
        ptx::mbar_expect_tx(&full_bar[s], C::kTxBytes);
        ptx::tma_load_3d(sa, &tmA, &full_bar[s], i * kBK, m0, 0);
        ptx::tma_load_3d(sa + C::kABytes, &tmB, &full_bar[s], i * kBK, n0, 0);
        bulk_g2s(sf, sfa_src + static_cast<long long>(i) * kSfChunk, kSfChunk, &full_bar[s]);
        bulk_g2s(sf + kSfChunk, sfb_src + static_cast<long long>(i) * kSfChunk, kSfChunk, &full_bar[s]);
      }
      __syncwarp();
    }
  } else if (warp < 4) {
    float acc0[BN / 2], acc1[BN / 2], part[BN / 2];
    wg::zero(acc0);
    wg::zero(acc1);
    const int b_col0 = n0 & 127;   // chunk row of the tile's first B row
    uint8_t* wa = smem + C::kWideOff;
    uint8_t* wb = wa + C::kWideA;
    const uint32_t wa_u = ptx::smem_u32(wa), wb_u = ptx::smem_u32(wb);
    for (int i = 0; i < n_kb; ++i) {
      const int s = i % C::kStages;
      const uint32_t ph = (i / C::kStages) & 1;
      ptx::mbar_wait(&full_bar[s], ph);
      const uint8_t* st = smem + s * C::kTileStage;
      const uint8_t* sf = smem + C::kSfOff + s * C::kSfStage;
      // every thread's wgmma of the previous K-block retired before the f16 copies are rewritten
      asm volatile("bar.sync 2, 128;" ::: "memory");
      wg::widen_e4m3_tile(wa, st, kBM, threadIdx.x, 128);
      wg::widen_e4m3_tile(wb, st + C::kABytes, BN, threadIdx.x, 128);
      ptx::fence_proxy_async_smem();
      asm volatile("bar.sync 2, 128;" ::: "memory");
#pragma unroll
      for (int g = 0; g < 4; ++g) {     // K-group g: elements 32g .. 32g+31 = f16 tile g / 2, 64 bytes in
        const uint32_t ko = (g & 1) * 64u;
#pragma unroll
        for (int h = 0; h < 2; ++h) {   // rows 64h .. 64h+63
          const uint32_t a0 = wa_u + (g >> 1) * (kBM * 128u) + h * 8192u + ko;
          const uint32_t b0 = wb_u + (g >> 1) * (BN * 128u) + ko;
          wg::fence();
          wg::wgmma_f16_n64(part, wg::desc(a0, 16), wg::desc(b0, 16), 0u);
          wg::wgmma_f16_n64(part, wg::desc(a0 + 32u, 16), wg::desc(b0 + 32u, 16), 1u);
          wg::commit();
          wg::wait<0>();
          wg::reg_fence(part);
          if (h == 0) wg::mx_accumulate<BN>(acc0, part, sf, 0, sf + kSfChunk, b_col0, g);
          else wg::mx_accumulate<BN>(acc1, part, sf, 64, sf + kSfChunk, b_col0, g);
        }
      }
      ptx::mbar_arrive(&empty_bar[s]);
    }
    wg::acc_put<BN>(at, 0, acc0, [](int r) { return r; });
    wg::acc_put<BN>(at, 0, acc1, [](int r) { return 64 + r; });
    ptx::mbar_arrive(accum_bar);
  } else {
    const int q = warp & 3;
    float* stg = stage_base + (warp - kEpiWarp0) * (32 * kStgLd);
    const int row_base = m0 + q * 32;
    const int cr = lane >> 3, cg = (lane & 7) * 4;
    {
      const int et = threadIdx.x - kEpiWarp0 * 32;
      for (int i = et; i < BN; i += 128)
        sbias[i] = (p.bias != nullptr && n0 + i < p.N) ? __ldg(p.bias + n0 + i) : 0.f;
      asm volatile("bar.sync 1, 128;" ::: "memory");
    }
    ptx::mbar_wait(accum_bar, 0);
    const uint32_t taddr = static_cast<uint32_t>(q * 32) << 16;
#pragma unroll 1
    for (int c = 0; c < BN / 32; ++c) {
      const int nc = n0 + c * 32;
      if (nc >= p.N) break;
      uint32_t r[32];
      wg::acc_ld32(at, taddr + c * 32, r);
      float4* rowp = reinterpret_cast<float4*>(stg + lane * kStgLd);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float x = __uint_as_float(r[4 * j + k]) * p.alpha + sbias[c * 32 + 4 * j + k];
          if (p.act == 1) x = fmaxf(x, 0.f);
          else if (p.act == 2) x = gelu_f(x);
          v[k] = x;
        }
        rowp[j] = make_float4(v[0], v[1], v[2], v[3]);
      }
      __syncwarp();
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int rr = it * 4 + cr, rw = row_base + rr, col = nc + cg;
        if (rw >= p.M || col >= p.N) continue;
        const float4 x = *reinterpret_cast<const float4*>(stg + rr * kStgLd + cg);
        const long long off = static_cast<long long>(rw) * p.ldd + col;
        const bool vec = col + 3 < p.N;
        if (p.d_dtype == 0) {
          float* d = reinterpret_cast<float*>(p.d) + off;
          if (vec) *reinterpret_cast<float4*>(d) = x;
          else {
            const float xs[4] = {x.x, x.y, x.z, x.w};
            for (int k = 0; k < 4; ++k) if (col + k < p.N) d[k] = xs[k];
          }
        } else {
          __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(p.d) + off;
          if (vec) *reinterpret_cast<uint2*>(d) = make_uint2(pack2(x.x, x.y), pack2(x.z, x.w));
          else {
            const float xs[4] = {x.x, x.y, x.z, x.w};
            for (int k = 0; k < 4; ++k) if (col + k < p.N) d[k] = __float2bfloat16(xs[k]);
          }
        }
      }
      __syncwarp();
    }
  }
}

// ------------------------------------------------------------------ quantiser
template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f<uint8_t>(uint8_t v) { return static_cast<float>(v); }

// One thread per (row, 32-element K group) of the PADDED problem (rows to a multiple of 128,
// groups to a multiple of 4): amax -> UE8M0 exponent e, the smallest with 448 * 2^e >= amax
// (epi::mx8_scale_byte) -> e4m3 satfinite(x * 2^-e).  Padding groups / rows get scale 1.0 (0x7F;
// never NaN) and no data.
template <typename T>
__global__ void __launch_bounds__(256)
k_quantize_mx8(const T* __restrict__ x, long long ldx, int R, int K, float in_scale,
               uint8_t* __restrict__ q, long long ldq, uint8_t* __restrict__ sf, int k_blocks) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  const int groups = k_blocks * 4;
  const long long gid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const int row = static_cast<int>(gid / groups), g = static_cast<int>(gid % groups);
  const int r_pad = (R + 255) / 256 * 256;   // rows padded to 256 (the chunk array's fixed layout)
  if (row >= r_pad) return;
  const int r = row & 127, rb = row >> 7;
  uint8_t* sfp = sf + (static_cast<long long>(rb) * k_blocks + (g >> 2)) * kSfChunk + (r & 31) * 16 +
                 (r >> 5) * 4 + (g & 3);
  const int k0 = g * 32;
  if (row >= R || k0 >= K) { *sfp = 127; return; }
  const int n = min(32, K - k0);
  float v[32];
  const T* xp = x + static_cast<long long>(row) * ldx + k0;
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = i < n ? to_f<T>(xp[i]) * in_scale : 0.f;
  uint32_t w[8];
  *sfp = static_cast<uint8_t>(epi::mx8_quant32(v, w));
  // the row's bytes end at K rounded up to 16 (a wider pitch's tail belongs to the caller), so a
  // group is one or two 16-byte stores
  uint8_t* qp = q + static_cast<long long>(row) * ldq + k0;
  reinterpret_cast<uint4*>(qp)[0] = make_uint4(w[0], w[1], w[2], w[3]);
  if (n > 16) reinterpret_cast<uint4*>(qp)[1] = make_uint4(w[4], w[5], w[6], w[7]);
}

}  // namespace

cudaError_t gemm_mx8_sm100(const Mx8Problem& p, cudaStream_t stream) {
  bind_context_once();
  if (p.M <= 0 || p.N <= 0 || p.K <= 0 || p.ldd % 4 != 0 || p.lda % 16 != 0 || p.ldb % 16 != 0)
    return cudaErrorInvalidValue;
  const int mt = (p.M + kBM - 1) / kBM;
  constexpr int BN = 64;
  CUtensorMap ta, tb;
  GemmOperand oa{p.a, p.lda, 0, false}, ob{p.b, p.ldb, 0, false};
  cudaError_t e = gemm_make_operand_map(&ta, oa, DType::FP8_E4M3, p.M, p.K, 1, kBM);
  if (e != cudaSuccess) return e;
  e = gemm_make_operand_map(&tb, ob, DType::FP8_E4M3, p.N, p.K, 1, BN);
  if (e != cudaSuccess) return e;
  PM kp{};
  kp.M = p.M; kp.N = p.N; kp.K = p.K; kp.k_blocks = (p.K + kBK - 1) / kBK;
  kp.sfa = p.sfa; kp.sfb = p.sfb;
  kp.d = p.d; kp.d_dtype = static_cast<int>(p.d_dtype); kp.ldd = p.ldd; kp.alpha = p.alpha;
  kp.bias = p.bias; kp.act = static_cast<int>(p.act);
  dim3 grid(mt, (p.N + BN - 1) / BN, 1);
  note_launch();
  static bool cfg = false;
  if (!cfg) {
    e = cudaFuncSetAttribute(gemm_mx8_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<64>::kSmem);
    if (e != cudaSuccess) return e;
    cfg = true;
  }
  return launch_pdl(gemm_mx8_kernel<64>, grid, dim3(kThreads), Cfg<64>::kSmem, stream, ta, tb, kp);
}

long long mx8_sf_bytes(int rows, int K) {
  return static_cast<long long>((rows + 255) / 256 * 2) * ((K + kBK - 1) / kBK) * kSfChunk;
}

cudaError_t quantize_mx8(const void* x, DType x_dtype, long long ldx, int R, int K, float in_scale,
                         void* q, long long ldq, void* sf, cudaStream_t stream) {
  if (R <= 0 || K <= 0 || ldq % 16 != 0 || ldq < K) return cudaErrorInvalidValue;
  const int k_blocks = (K + kBK - 1) / kBK;
  const long long total = static_cast<long long>((R + 255) / 256 * 256) * k_blocks * 4;
  const dim3 grid(static_cast<unsigned>((total + 255) / 256)), block(256);
  uint8_t* q8 = static_cast<uint8_t*>(q);
  uint8_t* sf8 = static_cast<uint8_t*>(sf);
  note_launch();
  switch (x_dtype) {
    case DType::F32:
      return launch_pdl(k_quantize_mx8<float>, grid, block, 0, stream, static_cast<const float*>(x), ldx, R,
                        K, in_scale, q8, ldq, sf8, k_blocks);
    case DType::BF16:
      return launch_pdl(k_quantize_mx8<__nv_bfloat16>, grid, block, 0, stream,
                        static_cast<const __nv_bfloat16*>(x), ldx, R, K, in_scale, q8, ldq, sf8, k_blocks);
    case DType::U8:
      return launch_pdl(k_quantize_mx8<uint8_t>, grid, block, 0, stream, static_cast<const uint8_t*>(x), ldx,
                        R, K, in_scale, q8, ldq, sf8, k_blocks);
    default:
      return cudaErrorInvalidValue;
  }
}

}  // namespace bflc
