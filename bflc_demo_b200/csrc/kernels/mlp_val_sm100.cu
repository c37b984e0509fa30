// Committee validation of the 2-layer MLP: "QueryAllUpdates" + per-candidate scoring
// (reference: CommitteePrecompiled.cpp:299-311, python-sdk/main.py:196-217 -- one TF graph +
// Session per candidate there) as ONE launch:
//
//     fwd1 (K = in_dim, N = 256) -> +b1, relu -> A operand of fwd2 written straight from the
//     wgmma fragments into 128B-swizzled smem -> fwd2 (N = 64) -> +b2, argmax == label -> one
//     atomicAdd per warp into correct[z].  Warp 8 loads.
//
// One 2-CTA cluster per (64 rows, candidate z): each CTA computes half of the hidden layer and
// hands it to the leader through distributed shared memory, so even one candidate spreads over
// most of an H100's SMs.
//
// Candidate z's weights are addressed through device-resident tensor maps selected by the round
// plan (local staging slots filled by k_pull / k_pull_blob, or a trainer's upload buffer in peer
// HBM); inactive candidates exit.  Neither logits nor hidden activations ever reach global memory.
//
// One bf16 kernel serves both precisions.  In fp8 mode (MXFP8) the candidates travel as
// Mx8MlpLayout blobs (e4m3 weights + scale chunks + fp32 biases, 227 KB instead of 435 KB per
// candidate over NVLink), but the GEMMs read their exactly dequantised bf16 weights (the trainer's
// upload shadow, or the local staging slot k_pull_blob unpacks into) and x_dq, the exactly
// dequantised MXFP8 x: a bf16 wgmma with fp32 accumulation over those is the block-scaled product
// (epi::mx8_dq1).  Biases are fp32 from the blob (cand_blob[z]).
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

constexpr int kEpiWarps = 8;        // two MMA warpgroups
constexpr int kProducerWarp = kEpiWarps;
constexpr int kThreads = kEpiWarps * 32 + 32;
constexpr int kChainH = 256;
constexpr int kBarBytes = 512;
constexpr int kBiasFloats = 320;
constexpr int kBM = 64;
constexpr int kStages = 6;
constexpr int kA = kBM * 128, kB = 128 * 128, kStage = kA + kB;   // x 8 KB + this CTA's W1 half 16 KB
constexpr int kHalf = 2 * kBM * 128;        // 128 hidden columns of h: two 8 KB K-blocks of fwd2's A
constexpr int kOffH = kStages * kStage;     // h [64 x 256]: its own region, the peer's copy may land mid-fwd1
constexpr int kOffW2K = kOffH + 2 * kHalf;  // W2 K-major (leader only)
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

// One 2-CTA cluster per (64 validation rows, candidate z).  CTA rank r computes hidden columns
// 128 r .. 128 r + 127 of fwd1 for the 64 rows (MMA warpgroup g owns 64 of them: one m64n64k16
// per k16, so every hidden unit is one fp32 accumulation chain in K order), with one K-block of
// wgmma in flight.  relu(acc + b1) goes as bf16 into this CTA's half of the swizzled h tile; rank 1
// bulk-copies its half into the same offset of rank 0 (the leader), which completes the bytes on
// the leader's hx.  The leader alone loads W2 / b2 and runs fwd2 + argmax.  The final cluster
// barrier follows the leader's hx wait, so no CTA leaves while the copy reads or writes its smem.
// v is __grid_constant__: its fields are read where they are used, straight from the parameter
// bank, instead of all being loaded into registers at entry (61 registers instead of 62).
__global__ void __launch_bounds__(kThreads, 1)
mlp_val_pair_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ ValArgs v) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* empty = full + kStages;
  uint64_t* w2k = empty + kStages;
  uint64_t* hx = w2k + 1;
  float* sb = reinterpret_cast<float*>(smem + kOffBar + kBarBytes);

  ptx::pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = blockIdx.x & 1;   // clusters of 2 along x
  const bool leader = rank == 0;
  const int z = blockIdx.y, m0 = (blockIdx.x >> 1) * kBM;
  if (threadIdx.x == 0) {
    ptx::tma_prefetch_desc(&tmX);
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], kEpiWarps * 32);
    }
    ptx::mbar_init(w2k, 1);
    ptx::mbar_init(hx, 1);
    if (leader) ptx::mbar_expect_tx(hx, kHalf);   // the peer's half of h
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
      for (int kb = 0; kb < 4; ++kb) ptx::tma_load_3d(smem + kOffW2K + kb * 8192, m2, w2k, kb * 64, 0, 0);
    }
    __syncwarp();
    for (int i = 0; i < kb_d; ++i) {
      const int s = i % kStages;
      const uint32_t ph = (i / kStages) & 1;
      ptx::mbar_wait(&empty[s], ph ^ 1);
      if (ptx::elect_one()) {
        uint8_t* sa = smem + s * kStage;
        ptx::mbar_expect_tx(&full[s], kStage);
        ptx::tma_load_3d(sa, &tmX, &full[s], i * 64, m0, 0);
        ptx::tma_load_3d(sa + kA, m1, &full[s], i * 64, 128 * rank, 0);
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
      const int s = i % kStages;
      const uint32_t ph = (i / kStages) & 1;
      ptx::mbar_wait(&full[s], ph);
      const uint32_t sa = base + static_cast<uint32_t>(s) * kStage, sbw = sa + kA + g * 8192u;
      wg::fence();
#pragma unroll
      for (uint32_t k = 0; k < 4; ++k)
        wg::mma_bf16<64, 0, 0>(acc, wg::desc(sa + k * 32u, 16), wg::desc(sbw + k * 32u, 16),
                               (i > 0 || k > 0) ? 1u : 0u);
      wg::commit();
      wg::wait<1>();
      if (i > 0) ptx::mbar_arrive(&empty[(i - 1) % kStages]);
    }
    wg::wait<0>();
    wg::reg_fence(acc);
    asm volatile("bar.sync 1, 256;" ::: "memory");   // sb is loaded
    // ---- relu(acc + b1) -> K-block 2 rank + g of fwd2's A operand (swizzled smem)
    {
      const int c0 = 128 * static_cast<int>(rank) + 64 * g;
      uint8_t* tile = smem + kOffH + (c0 >> 6) * 8192;
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
        uint8_t* half = smem + kOffH + kHalf;
        ptx::bulk_s2cluster(ptx::mapa(ptx::smem_u32(half), 0), half, kHalf, ptx::mapa(ptx::smem_u32(hx), 0));
      }
    } else if (g == 0) {
      ptx::mbar_wait(hx, 0);    // the peer's half has landed
      ptx::mbar_wait(w2k, 0);
      // ---- fwd2: logits [64 x 64], K = 256
      float lg[32];
      wg::zero(lg);
      const uint32_t ha = base + kOffH, wb = base + kOffW2K;
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
  CUtensorMap tx;
  GemmOperand op{r.x, r.ldx, 0, false};
  cudaError_t e = gemm_make_operand_map(&tx, op, DType::BF16, r.n_val, r.in_dim, 1, kBM);
  if (e != cudaSuccess) return e;
  ValArgs v{};
  v.n_val = r.n_val; v.in_dim = r.in_dim; v.n_classes = r.n_classes;
  v.maps = r.maps; v.dyn1 = r.dyn1; v.dyn2 = r.dyn2;
  v.labels = r.labels; v.correct = r.correct;
  v.pred = r.pred ? r.pred : current_predicate();
  v.ql = mx8_mlp_layout(r.in_dim, r.hidden);
  if (r.fp8) v.cand_blob = r.cand_blob;
  static bool configured = false;
  if (!configured) {
    e = cudaFuncSetAttribute(mlp_val_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kValSmem);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  note_launch();
  const dim3 grid(2 * ((r.n_val + kBM - 1) / kBM), r.max_cand);
  return launch_pdl_cluster(2u, mlp_val_pair_kernel, grid, dim3(kThreads), kValSmem, stream, tx, v);
}

}  // namespace bflc
