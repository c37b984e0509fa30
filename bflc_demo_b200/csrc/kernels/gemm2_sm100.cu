// CTA-pair wgmma GEMM for large K-major bf16 problems on sm_90a -- persistent, one 2-CTA
// cluster per pair of SMs, the B tile shared between the two CTAs through TMA multicast.
//
// A cluster (2 x 1) computes one 256 x 256 output tile: CTA rank r owns rows [128 r, 128 r + 128)
// of it.  Per K-block (64 elements) each CTA loads its own 128 x 64 slice of A and HALF of the
// 256 x 64 B tile (rows [128 r, 128 r + 128)), multicast into the same smem offset of BOTH CTAs,
// so each SM pulls 32 KB out of L2 per K-block instead of the 48 KB of a 1-CTA 128 x 256 tile --
// the L2 -> SM feed is what bounds the single-CTA kernel on large problems.
//
//   warpgroup 0   TMA producer (one elected thread; setmaxnreg.dec to 40 registers)
//   warpgroups 1-2  consumers: rows [64 g, 64 g + 64) of the CTA's 128, m64n256k16 wgmma with the
//                 accumulator in registers (128 per thread; setmaxnreg.inc to 232), epilogue
//                 (alpha, bias, ReLU / GELU, fp32 or bf16 stores) straight from the fragments
//
// Stage hand-off: full[s] (local) completes when this CTA's A slice and both B halves have landed
// (48 KB of transactions, half of them issued by the peer); empty[s] collects one arrive per
// consumer warp of BOTH CTAs (the peer's warps arrive through the cluster address), because the
// producer's B half lands in the peer's stage s too.  Tiles are walked with a static stride over
// the clusters, M fastest so that clusters running at the same time share B tiles in L2; the
// producer runs ahead into the next tile while the consumers drain the epilogue of this one.
#include <cuda_bf16.h>

#include <cstring>

#include "bflc_kernels.h"
#include "epi_common.cuh"
#include "sm100_ptx.cuh"
#include "wgmma.cuh"

namespace bflc {

namespace {

constexpr int kBM = 128;           // rows per CTA (256 per cluster)
constexpr int kBN = 256;           // tile N (each CTA loads kBN / 2 rows of B)
constexpr int kStages = 4;
constexpr int kABytes = kBM * 128;           // 16 KB: 128 rows x 64 bf16
constexpr int kBHalf = (kBN / 2) * 128;      // 16 KB
constexpr int kStageBytes = kABytes + 2 * kBHalf;
constexpr int kThreads = 384;
constexpr int kConsumerWarps = 8;
constexpr int kSmemTotal = kStages * kStageBytes + 256 + 1024;
static_assert(kSmemTotal <= 227 * 1024, "shared memory budget");

struct P2 {
  int M, N, K, k_blocks, m_pairs, n_tiles;
  void* d; int d_dtype; long long ldd;
  float alpha; const float* bias; int act;
};

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// 3-D tiled load delivered to the same smem offset (and completing on the same mbarrier offset)
// in every CTA of `mask`
__device__ __forceinline__ void tma_load_3d_mc(void* smem_dst, const void* tmap, uint64_t* bar, int32_t c0,
                                               int32_t c1, int32_t c2, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster "
      "[%0], [%1, {%3, %4, %5}], [%2], %6;"
      :
      : "r"(ptx::smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(ptx::smem_u32(bar)),
        "r"(c0), "r"(c1), "r"(c2), "h"(mask)
      : "memory");
}
__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

__global__ void __launch_bounds__(kThreads, 1)
gemm2_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const P2 p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* empty = full + kStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = cluster_ctarank();
  const int cluster = blockIdx.x >> 1, n_clusters = gridDim.x >> 1;
  const int tiles = p.m_pairs * p.n_tiles;

  if (threadIdx.x == 0) {
    ptx::tma_prefetch_desc(&tmA);
    ptx::tma_prefetch_desc(&tmB);
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], 2 * kConsumerWarps);   // consumer warps of both CTAs
    }
    ptx::fence_mbar_init();
  }
  ptx::cluster_sync();   // both CTAs' barriers initialised before any multicast or remote arrive

  if (warp < 4) {
    // ------------------------------------------------------------------ producer warpgroup
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      uint32_t it = 0;
      for (int t = cluster; t < tiles; t += n_clusters) {
        const int m0 = (t % p.m_pairs) * 2 * kBM + static_cast<int>(rank) * kBM;
        const int n0 = (t / p.m_pairs) * kBN;
        for (int kb = 0; kb < p.k_blocks; ++kb, ++it) {
          const int s = it % kStages;
          ptx::mbar_wait(&empty[s], ((it / kStages) & 1) ^ 1);
          uint8_t* st = smem + s * kStageBytes;
          ptx::mbar_expect_tx(&full[s], kStageBytes);
          ptx::tma_load_3d(st, &tmA, &full[s], kb * 64, m0, 0);
          tma_load_3d_mc(st + kABytes + rank * kBHalf, &tmB, &full[s], kb * 64, n0 + static_cast<int>(rank) * (kBN / 2),
                         0, static_cast<uint16_t>(0x3));
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumer warpgroups
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int g = (warp >> 2) - 1;               // 0 | 1: rows [64 g, 64 g + 64) of the CTA's 128
    const int w = warp & 3;
    const uint32_t base = ptx::smem_u32(smem);
    uint32_t it = 0;
    float acc[kBN / 2];
    for (int t = cluster; t < tiles; t += n_clusters) {
      const int m0 = (t % p.m_pairs) * 2 * kBM + static_cast<int>(rank) * kBM;
      const int n0 = (t / p.m_pairs) * kBN;
      for (int kb = 0; kb < p.k_blocks; ++kb, ++it) {
        const int s = it % kStages;
        ptx::mbar_wait(&full[s], (it / kStages) & 1);
        const uint32_t sa = base + s * kStageBytes + g * 8192u, sb = base + s * kStageBytes + kABytes;
        wg::fence();
#pragma unroll
        for (uint32_t k = 0; k < 4; ++k)
          wg::mma_bf16<kBN, 0, 0>(acc, wg::desc(sa + k * 32u, 16), wg::desc(sb + k * 32u, 16), (kb > 0 || k > 0) ? 1u : 0u);
        wg::commit();
        // keep this K-block's group in flight; the previous one has retired -> release its stage
        wg::wait<1>();
        __syncwarp();
        if (kb > 0 && lane == 0) {
          const int sp = (it - 1) % kStages;
          ptx::mbar_arrive(&empty[sp]);
          ptx::mbar_arrive_cluster(&empty[sp], rank ^ 1u);
        }
      }
      wg::wait<0>();
      wg::reg_fence(acc);
      __syncwarp();
      if (p.k_blocks > 0 && lane == 0) {
        const int sp = (it - 1) % kStages;
        ptx::mbar_arrive(&empty[sp]);
        ptx::mbar_arrive_cluster(&empty[sp], rank ^ 1u);
      }
      // epilogue from the fragments: rows r0, r0 + 8; columns 8 j + 2 (lane % 4) + {0, 1}
      const int r0 = m0 + 64 * g + 16 * w + (lane >> 2);
#pragma unroll
      for (int i = 0; i < kBN / 2; i += 2) {
        const int row = r0 + 8 * ((i >> 1) & 1);
        const int col = n0 + wg::frag_col(i, lane);
        if (row >= p.M || col >= p.N) continue;
        float v[2] = {acc[i] * p.alpha, acc[i + 1] * p.alpha};
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          if (p.bias != nullptr && col + e < p.N) v[e] += __ldg(p.bias + col + e);
          if (p.act == 1) v[e] = fmaxf(v[e], 0.f);
          else if (p.act == 2) v[e] = gelu_f(v[e]);
        }
        const long long off = static_cast<long long>(row) * p.ldd + col;
        if (p.d_dtype == 0) {
          float* d = reinterpret_cast<float*>(p.d) + off;
          if (col + 1 < p.N) *reinterpret_cast<float2*>(d) = make_float2(v[0], v[1]);
          else d[0] = v[0];
        } else {
          __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(p.d) + off;
          if (col + 1 < p.N) *reinterpret_cast<uint32_t*>(d) = epi::pack_bf16x2(v[0], v[1]);
          else d[0] = __float2bfloat16(v[0]);
        }
      }
    }
  }
  // no CTA may leave while its peer can still multicast into it or arrive on its barriers
  ptx::cluster_sync();
}

}  // namespace

// D (M x N) = alpha * A (M x K, K-major) . B^T (N x K, K-major) [+ bias] [act]; ld % 4 == 0.
cudaError_t gemm2_sm100(const GemmProblem& p, cudaStream_t stream) {
  bind_context_once();
  if (p.ab_dtype != DType::BF16 || p.a.mn_major || p.b.mn_major || p.batch != 1 ||
      p.epi.kind != EpiKind::GENERIC || p.epi.split_k > 1 || p.epi.aux_in || p.epi.aux_out ||
      p.epi.colsum || p.epi.accumulate || p.epi.ldd % 4 != 0 || p.epi.d_dtype == DType::FP8_E4M3 ||
      p.b_maps_dev || p.dyn)
    return cudaErrorNotSupported;
  CUtensorMap ta, tb;
  cudaError_t e = gemm_make_operand_map(&ta, p.a, DType::BF16, p.M, p.K, 1, kBM);
  if (e != cudaSuccess) return e;
  e = gemm_make_operand_map(&tb, p.b, DType::BF16, p.N, p.K, 1, kBN / 2);
  if (e != cudaSuccess) return e;
  P2 kp{};
  kp.M = p.M; kp.N = p.N; kp.K = p.K; kp.k_blocks = (p.K + 63) / 64;
  kp.m_pairs = (p.M + 2 * kBM - 1) / (2 * kBM); kp.n_tiles = (p.N + kBN - 1) / kBN;
  kp.d = p.epi.d; kp.d_dtype = static_cast<int>(p.epi.d_dtype); kp.ldd = p.epi.ldd;
  kp.alpha = p.epi.alpha; kp.bias = p.epi.bias; kp.act = static_cast<int>(p.epi.act);
  static bool configured = false;
  static int max_clusters = 0;
  if (!configured) {
    e = cudaFuncSetAttribute(gemm2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotal);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(gemm2_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 0);
    (void)e;
    configured = true;
  }
  cudaLaunchConfig_t cfg{};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = kSmemTotal;
  cfg.stream = stream;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (max_clusters == 0) {
    // persistent: as many clusters as the device keeps resident at once (one CTA per SM)
    cfg.gridDim = dim3(2 * 1024);
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, gemm2_kernel, &cfg) != cudaSuccess || n <= 0) {
      (void)cudaGetLastError();
      int dev = 0, sms = 0;
      (void)cudaGetDevice(&dev);
      (void)cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
      n = sms / 2 > 0 ? sms / 2 : 1;
    }
    max_clusters = n;
  }
  const int tiles = kp.m_pairs * kp.n_tiles;
  const int clusters = tiles < max_clusters ? tiles : max_clusters;
  cfg.gridDim = dim3(2 * clusters, 1, 1);
  note_launch();
  return cudaLaunchKernelEx(&cfg, gemm2_kernel, ta, tb, kp);
}

}  // namespace bflc
