// Committee validation of the 2-layer MLP: "QueryAllUpdates" + per-candidate scoring
// (reference: CommitteePrecompiled.cpp:299-311, python-sdk/main.py:196-217 -- one TF graph +
// Session per candidate there) as ONE launch:
//
//     fwd1 (K = in_dim, N = 256) -> +b1, relu -> A operand of fwd2 written straight from the
//     wgmma fragments into 128B-swizzled smem -> fwd2 (N = 64) -> +b2, argmax == label -> one
//     atomicAdd per warp into correct[z].  Warp 8 loads.
//
// Two geometries.  mlp_val_pair_kernel (default): one 2-CTA cluster per (64 rows, candidate z),
// the hidden layer split between the pair and h handed to the leader through distributed shared
// memory -- 4x the CTAs of the 128-row kernel, which leaves most of an H100 idle at one
// candidate.  mlp_val_kernel: one CTA per (128 rows, candidate z), two MMA warpgroups of 64 rows
// each; the fused gather below runs on it, since its CTAs wait for each other's shares.
//
// Candidate z's weights are addressed through device-resident tensor maps selected by the round
// plan (local staging slots filled by k_pull, or a trainer's upload buffer in peer HBM); inactive
// candidates exit.  Neither logits nor hidden activations ever reach global memory.
//
// One bf16 kernel serves both precisions.  In fp8 mode (MXFP8) the candidates travel as
// Mx8MlpLayout blobs (e4m3 weights + scale chunks + fp32 biases, 227 KB instead of 435 KB per
// candidate over NVLink), but the GEMMs read their exactly dequantised bf16 weights (the trainer's
// upload shadow, or the local staging slot k_pull_blob / the fused gather below unpack into)
// and x_dq, the exactly dequantised MXFP8 x: a bf16 wgmma with fp32 accumulation over those is
// the block-scaled product (epi::mx8_dq1).  Biases are fp32 from the blob (cand_blob[z]).
#include <cuda_bf16.h>

#include <cstring>

#include "bflc_kernels.h"
#include "epi_common.cuh"
#include "launch.cuh"
#include "sm100_ptx.cuh"
#include "wgmma.cuh"

namespace bflc {

namespace {

__device__ __forceinline__ uint32_t pack2(float a, float b) { return epi::pack_bf16x2(a, b); }

constexpr int kBM = 128;
constexpr int kEpiWarps = 8;        // two MMA warpgroups
constexpr int kProducerWarp = kEpiWarps;
constexpr int kThreads = kEpiWarps * 32 + 32;
constexpr int kCStages = 3;
constexpr int kCA = kBM * 128, kCB = 256 * 128, kCStage = kCA + kCB;   // x tile 16 KB + W1 tile 32 KB
constexpr int kOffH = 0;                        // h tile (fwd2's A) aliases stage memory once fwd1 retired
constexpr int kOffW2K = kCStages * kCStage;     // W2 K-major, loaded up front
constexpr int kChainH = 256;
constexpr int kBarBytes = 512;
constexpr int kBiasFloats = 320;
constexpr int kOffBar = kOffW2K + 32768;
constexpr int kValSmem = kOffBar + kBarBytes + kBiasFloats * 4 + 1024;
static_assert(kValSmem <= 227 * 1024, "shared memory budget");

struct ValArgs {
  int n_val, in_dim, n_classes;
  const CUtensorMap* maps;               // table indexed by dyn{1,2}->map_index[z]
  const GemmDynamic* dyn1; const GemmDynamic* dyn2;
  const int32_t* labels; unsigned int* correct;
  const int* pred;
  // fp8: candidate z's blob (its fp32 biases), layout
  const uint8_t* const* cand_blob; Mx8MlpLayout ql;
  // fused gather of the candidate blobs (see MlpValArgs)
  const uint8_t* const* cand_src; unsigned int* pull_cnt;
  __nv_bfloat16* stage_dq; long long stage_stride; Mx8Unpack un;
  unsigned long long* stamps;
};

template <int R>
__device__ __forceinline__ void run_sync(float (&d)[R]) {
  wg::commit();
  wg::wait<0>();
  wg::reg_fence(d);
}

// b1 (all 256) and, when `with_b2`, b2 into sb: thread `et` of the two MMA warpgroups loads
// element et (kEpiWarps * 32 == kChainH)
__device__ __forceinline__ void load_biases(float* sb, const ValArgs& v, const uint8_t* blob, int z, bool with_b2) {
  const int et = threadIdx.x;
  const float* b1 = blob != nullptr ? reinterpret_cast<const float*>(blob + v.ql.b1) : v.dyn1->bias[z];
  sb[et] = b1 != nullptr ? b1[et] : 0.f;
  if (with_b2 && et < 64) {
    const float* b2 = blob != nullptr ? reinterpret_cast<const float*>(blob + v.ql.b2) : v.dyn2->bias[z];
    sb[kChainH + et] = (b2 != nullptr && et < v.n_classes) ? b2[et] : 0.f;
  }
}

// argmax over the C logits (+ b2) of fragment rows r0, r0 + 8 of one m64 tile at row m0 (first
// maximum wins) == label, one atomic per warp into correct[z]
__device__ __forceinline__ void score_rows(const float (&lg)[32], const float* sb, const ValArgs& v, int z,
                                           int m0, int r0) {
  const int lane = threadIdx.x & 31, C = v.n_classes;
  unsigned hits = 0;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    float vmax = -INFINITY;
    int amax = 0x7fffffff;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      if (((i >> 1) & 1) != e) continue;
      const int n = wg::frag_col(i, lane);
      const float x = lg[i] + sb[kChainH + n];
      if (n < C && (x > vmax || (x == vmax && n < amax))) { vmax = x; amax = n; }
    }
#pragma unroll
    for (int off = 1; off <= 2; off <<= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, vmax, off);
      const int oi = __shfl_xor_sync(0xffffffffu, amax, off);
      if (ov > vmax || (ov == vmax && oi < amax)) { vmax = ov; amax = oi; }
    }
    const int row = m0 + r0 + 8 * e;
    const bool hit = (lane & 3) == 0 && row < v.n_val && amax == v.labels[row];
    hits += __popc(__ballot_sync(0xffffffffu, hit));
  }
  if (lane == 0 && hits) atomicAdd(v.correct + z, hits);
}

__device__ __forceinline__ void val_stamp(unsigned long long* stamps, int slot) {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  atomicMax(stamps + slot, t);
}

__global__ void __launch_bounds__(kThreads, 1)
mlp_val_kernel(const __grid_constant__ CUtensorMap tmX, const ValArgs v) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* empty = full + kCStages;
  uint64_t* w2k = empty + kCStages;
  float* sb = reinterpret_cast<float*>(smem + kOffBar + kBarBytes);

  ptx::pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int z = blockIdx.y, m0 = blockIdx.x * kBM;
  if (warp == 0 && lane == 0) {
    ptx::tma_prefetch_desc(&tmX);
    for (int s = 0; s < kCStages; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], kEpiWarps * 32);
    }
    ptx::mbar_init(w2k, 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  ptx::pdl_wait();
  const bool inactive = (v.pred != nullptr && *v.pred == 0) || z >= v.dyn1->active_batches;
  if (inactive) return;
  const int kb_d = (v.in_dim + 63) / 64;
  const uint8_t* blob = v.cand_blob != nullptr ? v.cand_blob[z] : nullptr;

  if (v.cand_src != nullptr) {
    // ---- fused gather (reference: QueryAllUpdates, CommitteePrecompiled.cpp:299-311).  The
    // gridDim.x CTAs that validate candidate z each unpack 1/gridDim.x of z's blob out of the
    // trainer's HBM (P2P loads) as soon as its FLAG_TRAINED is up -- dequantised weights into the
    // local bf16 slot the B maps cover, biases into the local blob slot -- publish their share
    // (device-scope fence + counter), wait for the others' shares and only then start the TMA
    // loads of the local copy.  Every candidate crosses NVLink once per committee rank, and
    // there is no pull kernel in front of the validation.
    if (threadIdx.x == 0 && v.stamps != nullptr && blockIdx.x == 0 && z == 0) val_stamp(v.stamps, STAMP_PULL_BEGIN);
    if (threadIdx.x == 0 && v.dyn1->wait_flag[z] != nullptr)
      ptx::wait_flag_ge(v.dyn1->wait_flag[z], v.dyn1->wait_value);
    __syncthreads();
    const long long n = epi::mx8_unpack_units(v.un);
    const long long per = (n + gridDim.x - 1) / gridDim.x;
    const long long lo = per * blockIdx.x, hi = lo + per < n ? lo + per : n;
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x)
      epi::mx8_unpack_unit(v.un, v.cand_src[z], v.stage_dq + z * v.stage_stride, const_cast<uint8_t*>(blob), i);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      atomicAdd(v.pull_cnt + z, 1u);
      unsigned long long spins = 0;
      unsigned int have;
      do {
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(have) : "l"(v.pull_cnt + z) : "memory");
        if (have >= gridDim.x) break;
        __nanosleep(20);
      } while (++spins < (1ull << 26));
      if (have < gridDim.x) __trap();   // a sibling CTA never arrived: co-residency assumption broken
      if (v.stamps != nullptr && blockIdx.x == 0) val_stamp(v.stamps, STAMP_PULL_END);
    }
    __syncthreads();
    ptx::fence_proxy_async_all();   // the others' generic-proxy stores -> this CTA's TMA loads
  }

  if (warp == kProducerWarp) {
    if (v.dyn1->wait_flag[z] != nullptr) {   // candidate z's trainer has published its upload
      if (lane == 0) ptx::wait_flag_ge(v.dyn1->wait_flag[z], v.dyn1->wait_value);
      __syncwarp();
    }
    const CUtensorMap* m1 = v.maps + v.dyn1->map_index[z];
    const CUtensorMap* m2 = v.maps + v.dyn2->map_index[z];
    if (ptx::elect_one()) {
      ptx::mbar_expect_tx(w2k, 32768);
#pragma unroll
      for (int kb = 0; kb < 4; ++kb) ptx::tma_load_3d(smem + kOffW2K + kb * 8192, m2, w2k, kb * 64, 0, 0);
    }
    __syncwarp();
    for (int i = 0; i < kb_d; ++i) {
      const int s = i % kCStages;
      const uint32_t ph = (i / kCStages) & 1;
      ptx::mbar_wait(&empty[s], ph ^ 1);
      if (ptx::elect_one()) {
        uint8_t* sa = smem + s * kCStage;
        ptx::mbar_expect_tx(&full[s], kCStage);
        ptx::tma_load_3d(sa, &tmX, &full[s], i * 64, m0, 0);
        ptx::tma_load_3d(sa + kCA, m1, &full[s], i * 64, 0, 0);
      }
      __syncwarp();
    }
  } else if (warp < kEpiWarps) {
    // warpgroup g = rows 64g .. 64g+63 of the tile; thread rows r0 and r0 + 8
    const int g = warp >> 2, r0 = 64 * g + 16 * (warp & 3) + (lane >> 2);
    load_biases(sb, v, blob, z, true);
    const uint32_t base = ptx::smem_u32(smem);
    // ---- fwd1: [64 x 256] per warpgroup, K = in_dim
    float acc[4][32];   // four 64-column quarters of the 256 hidden units
#pragma unroll
    for (int t = 0; t < 4; ++t) wg::zero(acc[t]);
    for (int i = 0; i < kb_d; ++i) {
      const int s = i % kCStages;
      const uint32_t ph = (i / kCStages) & 1;
      ptx::mbar_wait(&full[s], ph);
      const uint32_t sa = base + static_cast<uint32_t>(s) * kCStage + g * 8192u, sbw = base + s * kCStage + kCA;
      wg::fence();
#pragma unroll
      for (uint32_t k = 0; k < 4; ++k)
#pragma unroll
        for (int t = 0; t < 4; ++t)
          wg::mma_bf16<64, 0, 0>(acc[t], wg::desc(sa + k * 32u, 16), wg::desc(sbw + t * 8192u + k * 32u, 16),
                                 (i > 0 || k > 0) ? 1u : 0u);
      wg::commit();
      wg::wait<0>();
#pragma unroll
      for (int t = 0; t < 4; ++t) wg::reg_fence(acc[t]);
      ptx::mbar_arrive(&empty[s]);
    }
    // every consumer is past its last stage read before h overwrites the ring (and sb is loaded)
    asm volatile("bar.sync 1, 256;" ::: "memory");
    // ---- relu(acc + b1) -> fwd2's A operand (swizzled smem), straight from the fragments
#pragma unroll
    for (int t = 0; t < 4; ++t) {
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int row = r0 + 8 * ((i >> 1) & 1), col = 64 * t + wg::frag_col(i, lane);
        uint8_t* tile = smem + kOffH + (col >> 6) * 16384 + row * 128;
        *reinterpret_cast<uint32_t*>(tile + ((((col & 63) >> 3) ^ (row & 7)) << 4) + (col & 7) * 2) =
            pack2(fmaxf(acc[t][i] + sb[col], 0.f), fmaxf(acc[t][i + 1] + sb[col + 1], 0.f));
      }
    }
    ptx::fence_proxy_async_smem();
    // fwd2 of this warpgroup reads only its own 64 rows of h
    if (g == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
    else asm volatile("bar.sync 3, 128;" ::: "memory");
    ptx::mbar_wait(w2k, 0);
    // ---- fwd2: logits [64 x 64], K = 256
    float lg[32];
    wg::zero(lg);
    const uint32_t ha = base + kOffH + g * 8192u, wb = base + kOffW2K;
    wg::fence();
#pragma unroll
    for (int kb = 0; kb < 4; ++kb)
#pragma unroll
      for (uint32_t k = 0; k < 4; ++k)
        wg::mma_bf16<64, 0, 0>(lg, wg::desc(ha + kb * 16384u + k * 32u, 16), wg::desc(wb + kb * 8192u + k * 32u, 16),
                               (kb > 0 || k > 0) ? 1u : 0u);
    run_sync(lg);
    score_rows(lg, sb, v, z, m0, r0);
  }
}

// ---- CTA-pair geometry (the default; see the file comment above mlp_val_pair_kernel)
constexpr int kPBM = 64;
constexpr int kPStages = 6;
constexpr int kPA = kPBM * 128, kPB = 128 * 128, kPStage = kPA + kPB;   // x 8 KB + this CTA's W1 half 16 KB
constexpr int kPHalf = 2 * kPBM * 128;          // 128 hidden columns of h: two 8 KB K-blocks of fwd2's A
constexpr int kPOffH = kPStages * kPStage;      // h [64 x 256]: its own region, the peer's copy may land mid-fwd1
constexpr int kPOffW2K = kPOffH + 2 * kPHalf;   // W2 K-major (leader only)
constexpr int kPOffBar = kPOffW2K + 32768;
constexpr int kPValSmem = kPOffBar + kBarBytes + kBiasFloats * 4 + 1024;
static_assert(kPValSmem <= 227 * 1024, "shared memory budget");

// One 2-CTA cluster per (64 validation rows, candidate z).  CTA rank r computes hidden columns
// 128 r .. 128 r + 127 of fwd1 for the 64 rows (MMA warpgroup g owns 64 of them: one m64n64k16
// per k16, the same accumulation chain per hidden unit as the 128-row kernel), with one K-block of
// wgmma in flight.  relu(acc + b1) goes as bf16 into this CTA's half of the swizzled h tile; rank 1
// bulk-copies its half into the same offset of rank 0 (the leader), which completes the bytes on
// the leader's hx.  The leader alone loads W2 / b2 and runs fwd2 + argmax.  The final cluster
// barrier follows the leader's hx wait, so no CTA leaves while the copy reads or writes its smem.
__global__ void __launch_bounds__(kThreads, 1)
mlp_val_pair_kernel(const __grid_constant__ CUtensorMap tmX, const ValArgs v) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kPOffBar);
  uint64_t* empty = full + kPStages;
  uint64_t* w2k = empty + kPStages;
  uint64_t* hx = w2k + 1;
  float* sb = reinterpret_cast<float*>(smem + kPOffBar + kBarBytes);

  ptx::pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = blockIdx.x & 1;   // clusters of 2 along x
  const bool leader = rank == 0;
  const int z = blockIdx.y, m0 = (blockIdx.x >> 1) * kPBM;
  if (threadIdx.x == 0) {
    ptx::tma_prefetch_desc(&tmX);
    for (int s = 0; s < kPStages; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], kEpiWarps * 32);
    }
    ptx::mbar_init(w2k, 1);
    ptx::mbar_init(hx, 1);
    if (leader) ptx::mbar_expect_tx(hx, kPHalf);   // the peer's half of h
    ptx::fence_mbar_init();
  }
  ptx::cluster_sync();   // both CTAs' mbarriers exist before any copy can target them
  ptx::pdl_wait();
  // the same for both CTAs of a pair (same z), so a pair exits or runs together
  const bool inactive = (v.pred != nullptr && *v.pred == 0) || z >= v.dyn1->active_batches;
  if (inactive) return;
  const int kb_d = (v.in_dim + 63) / 64;
  const uint8_t* blob = v.cand_blob != nullptr ? v.cand_blob[z] : nullptr;

  if (warp == kProducerWarp) {
    if (v.dyn1->wait_flag[z] != nullptr) {   // candidate z's trainer has published its upload
      if (lane == 0) ptx::wait_flag_ge(v.dyn1->wait_flag[z], v.dyn1->wait_value);
      __syncwarp();
    }
    const CUtensorMap* m1 = v.maps + v.dyn1->map_index[z];
    const CUtensorMap* m2 = v.maps + v.dyn2->map_index[z];
    if (leader && ptx::elect_one()) {
      ptx::mbar_expect_tx(w2k, 32768);
#pragma unroll
      for (int kb = 0; kb < 4; ++kb) ptx::tma_load_3d(smem + kPOffW2K + kb * 8192, m2, w2k, kb * 64, 0, 0);
    }
    __syncwarp();
    for (int i = 0; i < kb_d; ++i) {
      const int s = i % kPStages;
      const uint32_t ph = (i / kPStages) & 1;
      ptx::mbar_wait(&empty[s], ph ^ 1);
      if (ptx::elect_one()) {
        uint8_t* sa = smem + s * kPStage;
        ptx::mbar_expect_tx(&full[s], kPStage);
        ptx::tma_load_3d(sa, &tmX, &full[s], i * 64, m0, 0);
        ptx::tma_load_3d(sa + kPA, m1, &full[s], i * 64, 128 * rank, 0);
      }
      __syncwarp();
    }
  } else if (warp < kEpiWarps) {
    // warpgroup g = hidden columns 128 rank + 64 g .. +63; thread rows r0 and r0 + 8
    const int g = warp >> 2, r0 = 16 * (warp & 3) + (lane >> 2);
    load_biases(sb, v, blob, z, leader);
    const uint32_t base = ptx::smem_u32(smem);
    // ---- fwd1: [64 x 64] per warpgroup, K = in_dim.  One K-block of wgmma stays in flight: a
    // stage is released once the next K-block's wait<1> shows that its wgmma have retired.
    float acc[32];
    wg::zero(acc);
    for (int i = 0; i < kb_d; ++i) {
      const int s = i % kPStages;
      const uint32_t ph = (i / kPStages) & 1;
      ptx::mbar_wait(&full[s], ph);
      const uint32_t sa = base + static_cast<uint32_t>(s) * kPStage, sbw = sa + kPA + g * 8192u;
      wg::fence();
#pragma unroll
      for (uint32_t k = 0; k < 4; ++k)
        wg::mma_bf16<64, 0, 0>(acc, wg::desc(sa + k * 32u, 16), wg::desc(sbw + k * 32u, 16),
                               (i > 0 || k > 0) ? 1u : 0u);
      wg::commit();
      wg::wait<1>();
      if (i > 0) ptx::mbar_arrive(&empty[(i - 1) % kPStages]);
    }
    wg::wait<0>();
    wg::reg_fence(acc);
    asm volatile("bar.sync 1, 256;" ::: "memory");   // sb is loaded
    // ---- relu(acc + b1) -> K-block 2 rank + g of fwd2's A operand (swizzled smem)
    {
      const int c0 = 128 * static_cast<int>(rank) + 64 * g;
      uint8_t* tile = smem + kPOffH + (c0 >> 6) * 8192;
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int row = r0 + 8 * ((i >> 1) & 1), col = wg::frag_col(i, lane);
        *reinterpret_cast<uint32_t*>(tile + row * 128 + (((col >> 3) ^ (row & 7)) << 4) + (col & 7) * 2) =
            pack2(fmaxf(acc[i] + sb[c0 + col], 0.f), fmaxf(acc[i + 1] + sb[c0 + col + 1], 0.f));
      }
    }
    ptx::fence_proxy_async_smem();
    asm volatile("bar.sync 1, 256;" ::: "memory");   // this CTA's half of h is written
    if (!leader) {
      if (threadIdx.x == 0) {
        uint8_t* half = smem + kPOffH + kPHalf;
        ptx::bulk_s2cluster(ptx::mapa(ptx::smem_u32(half), 0), half, kPHalf, ptx::mapa(ptx::smem_u32(hx), 0));
      }
    } else if (g == 0) {
      ptx::mbar_wait(hx, 0);    // the peer's half has landed
      ptx::mbar_wait(w2k, 0);
      // ---- fwd2: logits [64 x 64], K = 256
      float lg[32];
      wg::zero(lg);
      const uint32_t ha = base + kPOffH, wb = base + kPOffW2K;
      wg::fence();
#pragma unroll
      for (int kb = 0; kb < 4; ++kb)
#pragma unroll
        for (uint32_t k = 0; k < 4; ++k)
          wg::mma_bf16<64, 0, 0>(lg, wg::desc(ha + kb * 8192u + k * 32u, 16), wg::desc(wb + kb * 8192u + k * 32u, 16),
                                 (kb > 0 || k > 0) ? 1u : 0u);
      run_sync(lg);
      score_rows(lg, sb, v, z, m0, r0);
    }
  }
  __syncwarp();
  ptx::cluster_sync();
}

}  // namespace

cudaError_t mlp_val_sm100(const MlpValArgs& r, cudaStream_t stream) {
  bind_context_once();
  if (r.hidden != kChainH || r.n_classes > 64 || r.in_dim % 8 || r.n_val <= 0 || r.max_cand <= 0)
    return cudaErrorInvalidValue;
  if (r.fp8 && r.cand_blob == nullptr) return cudaErrorInvalidValue;
  // the fused gather's CTAs wait for each other, which needs the 128-row grid (see below)
  if (r.split && r.cand_src != nullptr) return cudaErrorInvalidValue;
  const int bm = r.split ? kPBM : kBM;
  CUtensorMap tx;
  GemmOperand op{r.x, r.ldx, 0, false};
  cudaError_t e = gemm_make_operand_map(&tx, op, DType::BF16, r.n_val, r.in_dim, 1, bm);
  if (e != cudaSuccess) return e;
  ValArgs v{};
  v.n_val = r.n_val; v.in_dim = r.in_dim; v.n_classes = r.n_classes;
  v.maps = r.maps; v.dyn1 = r.dyn1; v.dyn2 = r.dyn2;
  v.labels = r.labels; v.correct = r.correct;
  v.pred = r.pred ? r.pred : current_predicate();
  v.ql = mx8_mlp_layout(r.in_dim, r.hidden);
  if (r.fp8) v.cand_blob = r.cand_blob;
  if (r.cand_src != nullptr) {
    // every CTA of a candidate must be able to run while its siblings spin on the counter
    if (!r.fp8 || r.pull_cnt == nullptr || r.stage_dq == nullptr || r.in_dim % 16 != 0 ||
        (r.n_val + kBM - 1) / kBM > 128)
      return cudaErrorInvalidValue;
    v.cand_src = r.cand_src; v.pull_cnt = r.pull_cnt;
    v.stage_dq = static_cast<__nv_bfloat16*>(r.stage_dq); v.stage_stride = r.stage_stride;
    v.un = mx8_unpack_args(r.in_dim, r.hidden, r.n_classes, r.w1_off, r.w2_off);
    v.stamps = r.stamps;
  }
  if (r.split) {
    static bool configured_pair = false;
    if (!configured_pair) {
      e = cudaFuncSetAttribute(mlp_val_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPValSmem);
      if (e != cudaSuccess) return e;
      configured_pair = true;
    }
    note_launch();
    const dim3 grid(2 * ((r.n_val + kPBM - 1) / kPBM), r.max_cand);
    return launch_pdl_cluster(2u, mlp_val_pair_kernel, grid, dim3(kThreads), kPValSmem, stream, tx, v);
  }
  static bool configured = false;
  if (!configured) {
    e = cudaFuncSetAttribute(mlp_val_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kValSmem);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  note_launch();
  const dim3 grid((r.n_val + kBM - 1) / kBM, r.max_cand);
  return launch_pdl(mlp_val_kernel, grid, dim3(kThreads), kValSmem, stream, tx, v);
}

}  // namespace bflc
