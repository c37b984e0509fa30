// wgmma / TMA GEMM for sm_90a with fused epilogues.
//
//   D[b] (M x N) = alpha * A[b] (M x K) . B[b]^T (N x K)   bf16 or fp8(e4m3) in, fp32 accumulate
//
// One CTA computes one 128 x BN output tile (BN = 64 | 128):
//   warps 0-3: MMA warpgroup (two m64 x BN wgmma per K-step, accumulator in registers, parked
//              in a shared-memory accumulator tile when the reduction is done)
//   warp 4   : TMA producer  (cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier tx)
//   warps 5-8: epilogue (accumulator tile -> registers, one row per thread -> fused math -> global)
//
// Operands may be K-major or MN-major (transposed views), so forward (x.W^T),
// input-gradient (dY.W) and weight-gradient (dY^T.X) GEMMs all run without a transpose
// pass.  The B operand may come from a per-batch tensor-map array in device memory, whose
// maps may point into *peer GPUs'* HBM: the committee's validation GEMM pulls each
// trainer's candidate weights over NVLink tile by tile (hot path 1, X5 in SURVEY.md 2.7b).
//
// Epilogues: bias / ReLU / GELU / activation-backward masks / column sums (bias grads) /
// split-K atomics; a row-wise softmax-cross-entropy epilogue that emits dlogits + loss +
// #correct; an argmax-accuracy epilogue (the committee score, python-sdk/main.py:182-183).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <mutex>

#include "bflc_kernels.h"
#include "epi_common.cuh"
#include "launch.cuh"
#include "sm100_ptx.cuh"
#include "wgmma.cuh"

namespace bflc {

namespace {

constexpr int kBM = 128;             // two m64 wgmma per K-step
constexpr int kStageKBytes = 128;    // one swizzle-128B span of K per stage row
constexpr int kThreads = 288;
constexpr int kProducerWarp = 4, kEpiWarp0 = 5;
constexpr int kFp8Stages = 3;
constexpr int kABytes = kBM * kStageKBytes;  // 16 KB

struct KParams {
  int M, N, K, batch;
  int is_fp8;
  int a_mn, b_mn;           // 1 = MN-major
  int a_batched, b_batched;
  int k_blocks;             // total K blocks of BLOCK_K elements
  int split_k;
  const CUtensorMap* b_maps_dev;
  const GemmDynamic* dyn;
  const int* pred;
  long long* dbg_times;  // optional [8] clock64 stamps written by CTA (0,0,0) (bring-up only)
  // epilogue
  void* d;
  int d_dtype;
  long long ldd, d_batch_stride;
  float alpha;
  const float* bias;
  const float* const* bias_ptrs;
  int act;
  void* aux_out;
  const void* aux_in;
  int act_bwd;
  float* colsum;
  int accumulate;
  const int32_t* labels;
  long long labels_batch_stride;
  float grad_scale;
  float* loss_sum;
  unsigned int* correct;
  uint32_t lbo_a, sbo_a, lbo_b, sbo_b;
  uint32_t kstep_a, kstep_b;  // descriptor start-address advance per MMA K-step (bytes)
  int vec_ok;                 // d / aux rows are 16-byte aligned -> vectorised global access
  // implicit-GEMM convolution (ConvView): which operand is the shifted NHWC view and its taps
  int cv_mode, cv_flip;
  int cv_cb;                  // 64-channel blocks per filter tap
  int cv_kw, cv_pad, cv_stride;
  int cv_oh, cv_ow;           // pixel grid enumerated by the rows (mode 1) / the reduction (mode 2)
  int cv_c;                   // channels of the viewed activation
  int stages;                 // smem ring depth of this launch (<= SmemLayout::kStages)
  // EPI 3 (conv mode 2 by K groups, conv_dw_groups): grid z = group g, which reduces its own group_kb K
  // blocks [g group_kb, (g + 1) group_kb); pe_sq != nullptr: the epilogue squares and reduces the tile
  // into pe_sq[tile * groups + g], else it stores the fp32 tile into slice g of d (d_batch_stride apart)
  int group_kb;
  float* pe_sq;
};

template <int BN>
struct SmemLayout {
  static constexpr int kBBytes = BN * kStageKBytes;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = BN == 128 ? 4 : 6;
  static constexpr int kTileBytes = kStages * kStageBytes;
  static constexpr int kBarBytes = 256;
  static constexpr int kStgBytes = 4 * 32 * 36 * 4;  // per-epilogue-warp [32][36] fp32 staging
  static constexpr int kBiasBytes = BN * 4;
  static constexpr int kAccPitch = BN + 4;
  static constexpr int kAccBytes = kBM * kAccPitch * 4;   // fp32 accumulator tile
  static constexpr int kTotal = kTileBytes + kBarBytes + kStgBytes + kBiasBytes + kAccBytes + 1024;
  // e4m3 launches (BN = 64, kFp8Stages): f16 copies of the landed A and B stage after the tile
  static constexpr int kWideBytes = kBM * 256 + BN * 256 + 1024;   // + alignment
  static_assert(kTotal <= 227 * 1024, "shared memory budget");
};

using epi::kStgLd;
using epi::col_sum32;
using epi::stage_put;
using epi::stage_get;
using epi::pack_bf16x2;

// Staged [32][32] fp32 tile -> global.  Lane (cr, cg) moves 4 consecutive columns of row
// it*4+cr, so one warp instruction covers 4 rows x 128 B.  DT: 0 fp32, 1 bf16, 2 fp8(e4m3).
template <int DT, bool RED>
__device__ __forceinline__ void tile_store(const float* stg, void* dptr, long long tile_off,
                                           long long ldd, int row_base, int nc, int M, int N,
                                           int cr, int cg, int vec_ok) {
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int rr = it * 4 + cr;
    const int row = row_base + rr;
    const int col = nc + cg;
    if (row >= M || col >= N) continue;
    const float4 x = *reinterpret_cast<const float4*>(stg + rr * kStgLd + cg);
    const float xs[4] = {x.x, x.y, x.z, x.w};
    const long long off = tile_off + static_cast<long long>(row) * ldd + col;
    const bool vec = vec_ok && (col + 3 < N);
    if constexpr (DT == 0) {
      float* d = reinterpret_cast<float*>(dptr) + off;
      if constexpr (RED) {
        if (vec) ptx::red_add_f32x4(d, x.x, x.y, x.z, x.w);
        else
          for (int k = 0; k < 4; ++k) if (col + k < N) atomicAdd(d + k, xs[k]);
      } else {
        if (vec) *reinterpret_cast<float4*>(d) = x;
        else
          for (int k = 0; k < 4; ++k) if (col + k < N) d[k] = xs[k];
      }
    } else if constexpr (DT == 1) {
      __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(dptr) + off;
      if (vec) *reinterpret_cast<uint2*>(d) = make_uint2(pack_bf16x2(x.x, x.y), pack_bf16x2(x.z, x.w));
      else
        for (int k = 0; k < 4; ++k) if (col + k < N) d[k] = __float2bfloat16(xs[k]);
    } else {
      __nv_fp8_e4m3* d = reinterpret_cast<__nv_fp8_e4m3*>(dptr) + off;
      for (int k = 0; k < 4; ++k) if (col + k < N) d[k] = __nv_fp8_e4m3(xs[k]);
    }
  }
}
// global bf16 tile -> staged fp32 tile (zeros outside the matrix)
__device__ __forceinline__ void tile_load_bf16(float* stg, const void* sptr, long long tile_off,
                                               long long ldd, int row_base, int nc, int M, int N,
                                               int cr, int cg, int vec_ok) {
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int rr = it * 4 + cr;
    const int row = row_base + rr;
    const int col = nc + cg;
    float xs[4] = {0.f, 0.f, 0.f, 0.f};
    if (row < M && col < N) {
      const __nv_bfloat16* s = reinterpret_cast<const __nv_bfloat16*>(sptr) + tile_off +
                               static_cast<long long>(row) * ldd + col;
      if (vec_ok && col + 3 < N) {
        const uint2 u = *reinterpret_cast<const uint2*>(s);
        const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
        const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
        xs[0] = a.x; xs[1] = a.y; xs[2] = b.x; xs[3] = b.y;
      } else {
        for (int k = 0; k < 4; ++k) if (col + k < N) xs[k] = __bfloat162float(s[k]);
      }
    }
    *reinterpret_cast<float4*>(stg + rr * kStgLd + cg) = make_float4(xs[0], xs[1], xs[2], xs[3]);
  }
}

__device__ __forceinline__ float gelu_f(float x) {
  return 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
}
__device__ __forceinline__ float gelu_grad_f(float x) {
  const float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752f));
  const float pdf = 0.3989422804014327f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}

// The kernel body (KParams by value, as the kernels take it: existing instantiations compile to the
// same SASS as when this was the kernel itself).  kTail: after the main K blocks the producer loads one more stage from the
// low-rank tail maps (tmA2 / tmB2, the K2 <= 64 columns of A2 / B2 at K offset 0, zero-filled past
// K2 by TMA), so D = alpha * (A.B^T + A2.B2^T).  The tail pair has the main pair's majorness, so the
// MMA warpgroup's descriptors and the epilogue are the same; only the stage count grows by one.
template <int BN, int EPI, bool kTail>
__device__ __forceinline__ void gemm_body(const CUtensorMap& tmA, const CUtensorMap& tmB,
                                          const CUtensorMap& tmC, const KParams p,
                                          const CUtensorMap* tmA2, const CUtensorMap* tmB2) {
  using L = SmemLayout<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  // Ring depth is a launch parameter: short-K problems take a shallow ring so that two CTAs fit
  // one SM and one CTA's epilogue overlaps the other's main loop.
  const int n_stages = p.stages;
  const int tile_bytes = n_stages * L::kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + tile_bytes);
  uint64_t* empty_bar = full_bar + L::kStages;
  uint64_t* accum_bar = empty_bar + L::kStages;
  float* stage_base = reinterpret_cast<float*>(smem + tile_bytes + L::kBarBytes);
  float* sbias = stage_base + 4 * 32 * kStgLd;
  const wg::AccTile at{sbias + BN, L::kAccPitch};
  // e4m3 launches: f16 copies of the stage, 1024-aligned like every 128B-swizzled operand tile
  uint8_t* wide = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(at.p + kBM * L::kAccPitch) + 1023) & ~static_cast<uintptr_t>(1023));

  // Programmatic dependent launch: let the next kernel of the stream get scheduled now; this
  // CTA's own prologue (barrier init, descriptor prefetch) runs before it waits
  // for its predecessors' memory.
  ptx::pdl_launch_dependents();
  const long long t_entry = clock64();
  const bool dbg = p.dbg_times != nullptr && (blockIdx.x | blockIdx.y | blockIdx.z) == 0;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * BN;
  const int m0 = blockIdx.y * kBM;
  const int z = blockIdx.z;
  const int bidx = z / p.split_k;
  const int split = z - bidx * p.split_k;
  const int kb_per = EPI == 3 ? p.group_kb : (p.k_blocks + p.split_k - 1) / p.split_k;
  const int kb_begin = (EPI == 3 ? z : split) * kb_per;
  const int kb_end = min(p.k_blocks, kb_begin + kb_per);
  const int n_kb = max(0, kb_end - kb_begin);
  const int block_k = p.is_fp8 ? 128 : 64;  // elements per 128-byte span

  if (warp == 0 && lane == 0) {
    ptx::tma_prefetch_desc(&tmA);
    if (p.b_maps_dev == nullptr) ptx::tma_prefetch_desc(&tmB);
    if (p.cv_mode != 0) ptx::tma_prefetch_desc(&tmC);
    if constexpr (kTail) {
      ptx::tma_prefetch_desc(tmA2);
      ptx::tma_prefetch_desc(tmB2);
    }
    for (int s = 0; s < n_stages; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 128);   // every thread of the MMA warpgroup releases a slot
    }
    ptx::mbar_init(accum_bar, 128);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  if (dbg && threadIdx.x == 0) { p.dbg_times[0] = t_entry; p.dbg_times[1] = clock64(); }

  // Everything below touches memory produced by earlier kernels of the stream.
  ptx::pdl_wait();
  // role predication / dynamic batch count (device-resident, written by the plan kernel)
  const bool inactive = (p.pred != nullptr && *p.pred == 0) ||
                        (p.dyn != nullptr && bidx >= p.dyn->active_batches);
  if (inactive) return;  // CTA-uniform
  const CUtensorMap* mapB =
      p.b_maps_dev ? (p.b_maps_dev + (p.dyn ? p.dyn->map_index[bidx] : bidx)) : &tmB;

  if (warp == kProducerWarp) {
    // ------------------------------------------------------------ TMA producer
    // The whole warp runs the loop (warp-uniform control flow keeps addresses / coordinates in
    // uniform registers); one elected lane issues the copies.
    const int ca2 = p.a_batched ? bidx : 0;
    const int cb2 = (p.b_batched && !p.b_maps_dev) ? bidx : 0;
    if (p.dyn != nullptr && p.dyn->wait_flag[bidx] != nullptr) {
      // B lives in a peer's upload buffer: wait until that trainer released it, then make
      // the acquired state visible to the async proxy before the first TMA pull.
      if (lane == 0) ptx::wait_flag_ge(p.dyn->wait_flag[bidx], p.dyn->wait_value);
      __syncwarp();
      ptx::fence_proxy_async_all();
    }
    for (int i = 0; i < n_kb + (kTail ? 1 : 0); ++i) {
      const int s = i % n_stages;
      const uint32_t ph = (i / n_stages) & 1;
      ptx::mbar_wait(&empty_bar[s], ph ^ 1);
      uint8_t* sa = smem + s * L::kStageBytes;
      uint8_t* sb = sa + kABytes;
      int k0 = (kb_begin + i) * block_k;
      const CUtensorMap* mA = &tmA;
      const CUtensorMap* mB = mapB;
      if constexpr (kTail) {
        if (i == n_kb) { mA = tmA2; mB = tmB2; k0 = 0; }   // the low-rank tail stage
      }
      if (p.cv_mode != 0) {
        // ---- implicit-GEMM convolution: one operand is a tap-shifted NHWC box (tmC)
        if (ptx::elect_one()) {
          ptx::mbar_expect_tx(&full_bar[s], L::kStageBytes);
          const int kb = kb_begin + i;
          const int per_img = p.cv_oh * p.cv_ow;
          if (p.cv_mode == 1) {
            // rows m0.. = 128 consecutive output pixels (whole image rows); K block = (tap, 64 ch)
            const int tap = kb / p.cv_cb, cblk = kb - tap * p.cv_cb;
            const int r = tap / p.cv_kw, t = tap - r * p.cv_kw;
            const int img0 = m0 / per_img, oh0 = (m0 - img0 * per_img) / p.cv_ow;
            const int dh = p.cv_flip ? p.cv_pad - r : r - p.cv_pad;
            const int dw = p.cv_flip ? p.cv_pad - t : t - p.cv_pad;
            ptx::tma_load_4d(sa, &tmC, &full_bar[s], cblk * 64, dw, oh0 * p.cv_stride + dh, img0);
            if (!p.cv_flip) {
              ptx::tma_load_3d(sb, mapB, &full_bar[s], k0, n0, 0);
            } else {  // w[Cout][taps*Cin] read MN-major: N offset selects the tap, K = out channels
              for (int b = 0; b < BN / 64; ++b)
                ptx::tma_load_3d(sb + b * (64 * 128), mapB, &full_bar[s],
                                 tap * p.N + n0 + b * 64, cblk * 64, 0);
            }
          } else {
            // weight gradient: K block = 64 output pixels; N tile = (tap, BN channels)
            for (int b = 0; b < 2; ++b)  // A = dy^T, MN-major: two 64-wide boxes of out channels
              ptx::tma_load_3d(sa + b * (64 * 128), &tmA, &full_bar[s], m0 + b * 64, k0, 0);
            const int tap = n0 / p.cv_c, c0 = n0 - tap * p.cv_c;
            const int r = tap / p.cv_kw, t = tap - r * p.cv_kw;
            const int pix0 = kb * 64;
            const int img0 = pix0 / per_img, oh0 = (pix0 - img0 * per_img) / p.cv_ow;
            for (int b = 0; b < BN / 64; ++b)
              ptx::tma_load_4d(sb + b * (64 * 128), &tmC, &full_bar[s], c0 + b * 64, t - p.cv_pad,
                               oh0 * p.cv_stride + r - p.cv_pad, img0);
          }
        }
        __syncwarp();
        continue;
      }
      if (ptx::elect_one()) {
        ptx::mbar_expect_tx(&full_bar[s], L::kStageBytes);
        if (!p.a_mn) {
          ptx::tma_load_3d(sa, mA, &full_bar[s], k0, m0, ca2);
        } else {
          // MN-major: boxes of [block_k rows of K][128 B of M]; kBM*es/128 boxes
          const int nbox = p.is_fp8 ? 1 : 2;
          for (int b = 0; b < nbox; ++b)
            ptx::tma_load_3d(sa + b * (block_k * 128), mA, &full_bar[s], m0 + b * block_k, k0,
                             ca2);
        }
        if (!p.b_mn) {
          ptx::tma_load_3d(sb, mB, &full_bar[s], k0, n0, cb2);
        } else {
          const int nbox = BN / block_k;
          for (int b = 0; b < nbox; ++b)
            ptx::tma_load_3d(sb + b * (block_k * 128), mB, &full_bar[s], n0 + b * block_k, k0,
                             cb2);
        }
        if (dbg && i == 0) p.dbg_times[2] = clock64();
      }
      __syncwarp();
    }
  } else if (warp < 4) {
    // ------------------------------------------------------------- MMA warpgroup
    // Rows 0-63 and 64-127 of the tile are two m64 wgmma sharing the B descriptor; the A half
    // lives 8 KB further (64 K-major rows, or the second 64-wide box of an MN-major A).
    float acc0[BN / 2], acc1[BN / 2];
    wg::zero(acc0);
    wg::zero(acc1);
    const uint32_t base = ptx::smem_u32(smem);
    const bool fp8 = p.is_fp8 != 0;
    if (fp8) {
      // e4m3 operands widened to f16 per stage (exact), then f16 wgmma: its accumulation is full
      // fp32, the e4m3 wgmma's is not (wgmma.cuh, widen_e4m3_tile).  BN == 64 here.
      uint8_t* wa = wide;
      uint8_t* wb = wide + kBM * 256;
      const uint32_t wa_u = ptx::smem_u32(wa), wb_u = ptx::smem_u32(wb);
      for (int i = 0; i < n_kb; ++i) {
        const int s = i % n_stages;
        const uint32_t ph = (i / n_stages) & 1;
        ptx::mbar_wait(&full_bar[s], ph);
        const uint8_t* st = smem + s * L::kStageBytes;
        asm volatile("bar.sync 2, 128;" ::: "memory");   // previous K-block's wgmma retired everywhere
        wg::widen_e4m3_tile(wa, st, kBM, threadIdx.x, 128);
        wg::widen_e4m3_tile(wb, st + kABytes, BN, threadIdx.x, 128);
        ptx::mbar_arrive(&empty_bar[s]);
        ptx::fence_proxy_async_smem();
        asm volatile("bar.sync 2, 128;" ::: "memory");
        if constexpr (BN == 64) {
          wg::fence();
#pragma unroll
          for (uint32_t k = 0; k < 8; ++k) {   // 128 K-elements = two f16 tiles of 4 K-steps
            const uint32_t off = (k & 3u) * 32u;
            const uint64_t bd = wg::desc(wb_u + (k >> 2) * (BN * 128u) + off, 16);
            const uint32_t acc = (i > 0 || k > 0) ? 1u : 0u;
            wg::wgmma_f16_n64(acc0, wg::desc(wa_u + (k >> 2) * (kBM * 128u) + off, 16), bd, acc);
            wg::wgmma_f16_n64(acc1, wg::desc(wa_u + (k >> 2) * (kBM * 128u) + 8192u + off, 16), bd, acc);
          }
          wg::commit();
          wg::wait<0>();
          wg::reg_fence(acc0);
          wg::reg_fence(acc1);
        }
      }
    }
    for (int i = 0; i < (fp8 ? 0 : n_kb + (kTail ? 1 : 0)); ++i) {
      const int s = i % n_stages;
      const uint32_t ph = (i / n_stages) & 1;
      ptx::mbar_wait(&full_bar[s], ph);
      if (dbg && threadIdx.x == 0 && i == 0) p.dbg_times[3] = clock64();
      const uint32_t sa = base + static_cast<uint32_t>(s) * L::kStageBytes, sb = sa + kABytes;
      wg::fence();
#pragma unroll
      for (uint32_t k = 0; k < 4; ++k) {  // 4 K-steps (32 bytes of K) per 128-byte stage
        const uint64_t a0 = wg::desc(sa + k * p.kstep_a, p.lbo_a, p.sbo_a);
        const uint64_t a1 = wg::desc(sa + 8192u + k * p.kstep_a, p.lbo_a, p.sbo_a);
        const uint64_t bd = wg::desc(sb + k * p.kstep_b, p.lbo_b, p.sbo_b);
        const uint32_t acc = (i > 0 || k > 0) ? 1u : 0u;
        wg::mma_bf16_rt<BN>(acc0, a0, bd, acc, p.a_mn, p.b_mn);
        wg::mma_bf16_rt<BN>(acc1, a1, bd, acc, p.a_mn, p.b_mn);
      }
      wg::commit();
      wg::wait<0>();
      wg::reg_fence(acc0);
      wg::reg_fence(acc1);
      ptx::mbar_arrive(&empty_bar[s]);  // this thread's reads of the slot have retired
    }
    wg::acc_put<BN>(at, 0, acc0, [](int r) { return r; });
    wg::acc_put<BN>(at, 0, acc1, [](int r) { return 64 + r; });
    ptx::mbar_arrive(accum_bar);  // accumulator complete
    if (dbg && threadIdx.x == 0) p.dbg_times[4] = clock64();
  } else {

    // --------------------------------------------------------------- epilogue
    // accumulator tile -> registers (thread = one row) -> fused math -> per-warp smem staging
    // tile [32 rows][36 floats] -> global, so that every global instruction touches full
    // 128-byte lines (4 rows x 128 B per warp instruction) instead of 32 scattered rows.
    const int q = warp & 3;           // row quarter of the tile
    const int ew = warp - kEpiWarp0;  // epilogue warp index 0..3 (staging buffer owner)
    const int row_base = m0 + q * 32;
    const int row = row_base + lane;
    const bool row_ok = row < p.M;
    float* stg = stage_base + ew * (32 * kStgLd);
    const float* bias = p.dyn ? p.dyn->bias[bidx] : (p.bias_ptrs ? p.bias_ptrs[bidx] : p.bias);
    {  // bias tile -> smem once per CTA (coalesced), shared by the four epilogue warps
      const int et = threadIdx.x - kEpiWarp0 * 32;
      for (int i = et; i < BN; i += 128)
        sbias[i] = (bias != nullptr && n0 + i < p.N && split == 0) ? __ldg(bias + n0 + i) : 0.f;
      asm volatile("bar.sync 1, 128;" ::: "memory");
    }
    ptx::mbar_wait(accum_bar, 0);
    if (dbg && warp == kEpiWarp0 && lane == 0) p.dbg_times[5] = clock64();
    const uint32_t taddr = static_cast<uint32_t>(q * 32) << 16;
    const bool have_acc = n_kb > 0;
    const long long tile_off = static_cast<long long>(bidx) * p.d_batch_stride;
    // coalesced-phase coordinates of this lane: 4 rows x 8 column groups per instruction
    const int cr = lane >> 3, cg = (lane & 7) * 4;

    if constexpr (EPI == 3) {
      // one K group's tile: squared and reduced to one partial (fixed order: each row's columns in
      // order, the warp's butterfly, then the four warps in order), or stored into the group's slice
      float sq = 0.f;
#pragma unroll 1
      for (int c = 0; c < BN / 32; ++c) {
        const int nc = n0 + c * 32;
        if (nc >= p.N) break;  // warp-uniform
        uint32_t r[32];
        wg::acc_ld32(at, taddr + c * 32, r);
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = have_acc ? __uint_as_float(r[j]) : 0.f;
        if (p.pe_sq != nullptr) {
#pragma unroll
          for (int j = 0; j < 32; ++j) sq = fmaf(v[j], v[j], sq);
        } else {
          stage_put(stg, lane, v);
          __syncwarp();
          tile_store<0, false>(stg, p.d, tile_off, p.ldd, row_base, nc, p.M, p.N, cr, cg, p.vec_ok);
          __syncwarp();
        }
      }
      if (p.pe_sq != nullptr) {
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, off);
        if (lane == 0) stg[0] = sq;
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (warp == kEpiWarp0 && lane == 0) {
          float t = stage_base[0];
          for (int k = 1; k < 4; ++k) t += stage_base[k * 32 * kStgLd];
          p.pe_sq[static_cast<long long>(blockIdx.y * gridDim.x + blockIdx.x) * gridDim.z + z] = t;
        }
      }
    } else if constexpr (EPI == 0) {
#pragma unroll 1
      for (int c = 0; c < BN / 32; ++c) {
        const int nc = n0 + c * 32;
        if (nc >= p.N) break;  // warp-uniform
        uint32_t r[32];
        wg::acc_ld32(at, taddr + c * 32, r);
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j)
          v[j] = (have_acc ? __uint_as_float(r[j]) * p.alpha : 0.f) + sbias[c * 32 + j];
        if (p.aux_out != nullptr) {
          stage_put(stg, lane, v);
          __syncwarp();
          tile_store<1, false>(stg, p.aux_out, tile_off, p.ldd, row_base, nc, p.M, p.N, cr, cg,
                               p.vec_ok);
          __syncwarp();
        }
        if (p.act == 1) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
        } else if (p.act == 2) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = gelu_f(v[j]);
        }
        if (p.act_bwd != 0) {
          tile_load_bf16(stg, p.aux_in, tile_off, p.ldd, row_base, nc, p.M, p.N, cr, cg, p.vec_ok);
          __syncwarp();
          float a[32];
          stage_get(stg, lane, a);
          __syncwarp();
#pragma unroll
          for (int j = 0; j < 32; ++j)
            v[j] = (p.act_bwd == 1) ? (a[j] > 0.f ? v[j] : 0.f) : v[j] * gelu_grad_f(a[j]);
        }
        stage_put(stg, lane, v);
        __syncwarp();
        if (p.split_k > 1)
          tile_store<0, true>(stg, p.d, tile_off, p.ldd, row_base, nc, p.M, p.N, cr, cg, p.vec_ok);
        else if (p.d_dtype == 0)
          // d += tile: one writer per element, so a fire-and-forget red.add is deterministic and
          // has no load round trip (the read-modify-write form spent 32 dependent L2 latencies,
          // 16 us, in a 128 x 128 weight-gradient tile)
          (p.accumulate ? tile_store<0, true>(stg, p.d, tile_off, p.ldd, row_base, nc, p.M, p.N, cr,
                                              cg, p.vec_ok)
                        : tile_store<0, false>(stg, p.d, tile_off, p.ldd, row_base, nc, p.M, p.N,
                                               cr, cg, p.vec_ok));
        else if (p.d_dtype == 1)
          tile_store<1, false>(stg, p.d, tile_off, p.ldd, row_base, nc, p.M, p.N, cr, cg, p.vec_ok);
        else
          tile_store<2, false>(stg, p.d, tile_off, p.ldd, row_base, nc, p.M, p.N, cr, cg, p.vec_ok);
        if (p.colsum != nullptr) {
          // column sums straight from the staged tile: lane j adds up column j over valid rows
          const float tot = col_sum32(stg, lane, min(32, p.M - row_base));
          if (nc + lane < p.N) atomicAdd(p.colsum + nc + lane, tot);
        }
        __syncwarp();
      }
    } else {
      // ---------------- row-wise epilogues: the whole logit row lives in this CTA's tile
      const int32_t label =
          (row_ok && p.labels)
              ? p.labels[static_cast<long long>(bidx) * p.labels_batch_stride + row]
              : -1;
      // pass 1: max / argmax (+ label logit)
      float vmax = -INFINITY, zlab = 0.f;
      int amax = -1;
#pragma unroll 1
      for (int c = 0; c < BN / 32; ++c) {
        const int nc = c * 32;
        if (nc >= p.N) break;
        uint32_t r[32];
        wg::acc_ld32(at, taddr + c * 32, r);
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int n = nc + j;
          if (n < p.N) {
            const float x = __uint_as_float(r[j]) * p.alpha + sbias[n];
            if (x > vmax) { vmax = x; amax = n; }
            if (n == label) zlab = x;
          }
        }
      }
      const bool hit = row_ok && (amax == label);
      if constexpr (EPI == 2) {
        const unsigned cnt = __popc(__ballot_sync(0xffffffffu, hit));
        if (lane == 0 && cnt && p.correct) atomicAdd(p.correct + bidx, cnt);
      } else {
        // pass 2: sum exp
        float sum = 0.f;
#pragma unroll 1
        for (int c = 0; c < BN / 32; ++c) {
          const int nc = c * 32;
          if (nc >= p.N) break;
          uint32_t r[32];
          wg::acc_ld32(at, taddr + c * 32, r);
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const int n = nc + j;
            if (n < p.N) sum += __expf(__uint_as_float(r[j]) * p.alpha + sbias[n] - vmax);
          }
        }
        const float inv = 1.f / sum;
        float loss = row_ok ? (__logf(sum) + vmax - zlab) : 0.f;
        // pass 3: dlogits.  A dlogits row is ldd >= N columns wide and its pad columns [N, ldd)
        // get zeros; chunks that start at or past N read no accumulator (they may lie past the
        // BN-wide tile).  With ldd <= round_up(N, 32) this is the same chunk count as N alone.
        const int n_cols = p.d != nullptr ? static_cast<int>(p.ldd) : p.N;
#pragma unroll 1
        for (int nc = 0; nc < n_cols; nc += 32) {
          float v[32];
          if (nc < p.N) {  // warp-uniform
            uint32_t r[32];
            wg::acc_ld32(at, taddr + nc, r);
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              const int n = nc + j;
              float g = 0.f;
              if (n < p.N && row_ok) {
                const float x = __uint_as_float(r[j]) * p.alpha + sbias[n];
                g = (__expf(x - vmax) * inv - (n == label ? 1.f : 0.f)) * p.grad_scale;
              }
              v[j] = g;
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = 0.f;
          }
          stage_put(stg, lane, v);
          __syncwarp();
          if (p.d != nullptr)
            tile_store<1, false>(stg, p.d, tile_off, p.ldd, row_base, nc, p.M, n_cols, cr, cg,
                                 p.vec_ok);
          if (p.colsum != nullptr && nc < p.N) {
            const float tot = col_sum32(stg, lane, 32);
            if (nc + lane < p.N) atomicAdd(p.colsum + nc + lane, tot);
          }
          __syncwarp();
        }
        // loss / correct reductions
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, off);
        const unsigned cnt = __popc(__ballot_sync(0xffffffffu, hit));
        if (lane == 0) {
          if (p.loss_sum) atomicAdd(p.loss_sum, loss);
          if (p.correct && cnt) atomicAdd(p.correct + bidx, cnt);
        }
      }
    }
    if (dbg && warp == kEpiWarp0 && lane == 0) p.dbg_times[6] = clock64();
  }
  __syncthreads();
  if (dbg && threadIdx.x == 0) p.dbg_times[7] = clock64();
}

template <int BN, int EPI>
__global__ void __launch_bounds__(kThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tmC, const KParams p) {
  gemm_body<BN, EPI, false>(tmA, tmB, tmC, p, nullptr, nullptr);
}

// Generic epilogue with a low-rank K tail (LoRA linears: x.W^T + u.B^T, dz.W + v.A)
template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tail_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmC, const KParams p,
                 const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2) {
  gemm_body<BN, 0, true>(tmA, tmB, tmC, p, &tmA2, &tmB2);
}

// ------------------------------------------------------------------ host side
using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                              const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                              const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn get_encode() {
  static EncodeFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeFn>(sym);
  });
  return fn;
}

// rows_tile: number of M|N rows the CTA tile covers (128 for A, BN for B)
cudaError_t make_map(CUtensorMap* out, const GemmOperand& op, DType dt, int rows_extent, int K,
                     int batch, int rows_tile) {
  EncodeFn enc = get_encode();
  if (!enc) return cudaErrorNotSupported;
  const int es = (dt == DType::FP8_E4M3) ? 1 : 2;
  const int epb = 128 / es;  // elements per 128-byte swizzle span
  const CUtensorMapDataType cdt =
      (dt == DType::FP8_E4M3) ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  cuuint64_t dims[3], strides[2];
  cuuint32_t box[3], estr[3] = {1, 1, 1};
  const bool batched = op.batch_stride != 0 && batch > 1;
  if (!op.mn_major) {
    dims[0] = static_cast<cuuint64_t>(K);
    dims[1] = static_cast<cuuint64_t>(rows_extent);
    box[0] = epb;
    box[1] = static_cast<cuuint32_t>(rows_tile);
  } else {
    dims[0] = static_cast<cuuint64_t>(rows_extent);
    dims[1] = static_cast<cuuint64_t>(K);
    box[0] = epb;
    box[1] = epb;  // BLOCK_K rows of K
  }
  dims[2] = batched ? static_cast<cuuint64_t>(batch) : 1;
  box[2] = 1;
  strides[0] = static_cast<cuuint64_t>(op.ld) * es;
  strides[1] = batched ? static_cast<cuuint64_t>(op.batch_stride) * es
                       : strides[0] * dims[1];
  if ((strides[0] & 15) || (strides[1] & 15) || (reinterpret_cast<uintptr_t>(op.ptr) & 15))
    return cudaErrorMisalignedAddress;
  CUresult r = enc(out, cdt, 3, const_cast<void*>(op.ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    std::fprintf(stderr,
                 "[bflc] cuTensorMapEncodeTiled failed (CUresult %d): ptr=%p mn=%d dims={%llu,%llu,%llu} "
                 "strides={%llu,%llu} box={%u,%u,%u} es=%d\n",
                 static_cast<int>(r), op.ptr, op.mn_major ? 1 : 0,
                 static_cast<unsigned long long>(dims[0]), static_cast<unsigned long long>(dims[1]),
                 static_cast<unsigned long long>(dims[2]), static_cast<unsigned long long>(strides[0]),
                 static_cast<unsigned long long>(strides[1]), box[0], box[1], box[2], es);
    return cudaErrorInvalidValue;
  }
  return cudaSuccess;
}

// Pixel tile of `pix` output pixels as whole image rows: (pw, ph, pn) with pw*ph*pn == pix.
bool conv_pixel_tile(int pix, int OH, int OW, int* pw, int* ph, int* pn) {
  if (OW <= 0 || OH <= 0 || OW > pix || pix % OW != 0) return false;
  const int rows = pix / OW;
  if (rows <= OH) {
    if (OH % rows != 0) return false;
    *pw = OW; *ph = rows; *pn = 1;
  } else {
    if (rows % OH != 0) return false;
    *pw = OW; *ph = OH; *pn = rows / OH;
  }
  return true;
}

// 4-D map over an NHWC bf16 activation whose box is `pix` pixels x 64 channels, traversed with
// the convolution stride (elementStrides) so consecutive box rows are consecutive output pixels.
cudaError_t make_conv_map(CUtensorMap* out, const ConvView& cv, int pix) {
  EncodeFn enc = get_encode();
  if (!enc) return cudaErrorNotSupported;
  int pw, ph, pn;
  if (!conv_pixel_tile(pix, cv.OH, cv.OW, &pw, &ph, &pn)) return cudaErrorInvalidValue;
  if (cv.C % 64 != 0 || cv.stride < 1 || pw * cv.stride > 256 || ph * cv.stride > 256)
    return cudaErrorInvalidValue;
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(cv.C), static_cast<cuuint64_t>(cv.W),
                        static_cast<cuuint64_t>(cv.H), static_cast<cuuint64_t>(cv.N)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(cv.C) * 2,
                           static_cast<cuuint64_t>(cv.W) * cv.C * 2,
                           static_cast<cuuint64_t>(cv.H) * cv.W * cv.C * 2};
  cuuint32_t box[4] = {64, static_cast<cuuint32_t>(pw * cv.stride),
                       static_cast<cuuint32_t>(ph * cv.stride), static_cast<cuuint32_t>(pn)};
  cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(cv.stride), static_cast<cuuint32_t>(cv.stride), 1};
  if (reinterpret_cast<uintptr_t>(cv.x) & 15) return cudaErrorMisalignedAddress;
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(cv.x), dims, strides,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    std::fprintf(stderr, "[bflc] conv tensor map failed (CUresult %d): NHWC=%d,%d,%d,%d box=%u,%u,%u,%u stride=%d\n",
                 static_cast<int>(r), cv.N, cv.H, cv.W, cv.C, box[0], box[1], box[2], box[3], cv.stride);
    return cudaErrorInvalidValue;
  }
  return cudaSuccess;
}

template <int BN, int EPI>
cudaError_t launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc,
                   const KParams& kp, dim3 grid, cudaStream_t stream) {
  using L = SmemLayout<BN>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(gemm_kernel<BN, EPI>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  note_launch();
  const int smem = L::kTotal - (L::kStages - kp.stages) * L::kStageBytes + (kp.is_fp8 ? L::kWideBytes : 0);
  if (smem > L::kTotal) return cudaErrorInvalidValue;
  return launch_pdl(gemm_kernel<BN, EPI>, grid, dim3(kThreads), smem, stream, ta, tb, tc, kp);
}

template <int BN>
cudaError_t launch_tail(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc,
                        const KParams& kp, const CUtensorMap& ta2, const CUtensorMap& tb2,
                        dim3 grid, cudaStream_t stream) {
  using L = SmemLayout<BN>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(gemm_tail_kernel<BN>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  note_launch();
  const int smem = L::kTotal - (L::kStages - kp.stages) * L::kStageBytes;
  return launch_pdl(gemm_tail_kernel<BN>, grid, dim3(kThreads), smem, stream, ta, tb, tc, kp, ta2,
                    tb2);
}

}  // namespace

static unsigned long long g_launches = 0;
unsigned long long launch_count() { return g_launches; }
void note_launch() { ++g_launches; }
static thread_local long long* g_dbg_times = nullptr;
void set_debug_times(long long* p) { g_dbg_times = p; }
static bool g_pdl = true;
static unsigned long long g_pdl_fallbacks = 0;
void note_pdl_fallback() { ++g_pdl_fallbacks; }
unsigned long long pdl_fallbacks() { return g_pdl_fallbacks; }
void set_pdl(bool on) { g_pdl = on; }
bool pdl_enabled() { return g_pdl; }
static thread_local const int* g_pred = nullptr;
void set_predicate(const int* pred) { g_pred = pred; }
const int* current_predicate() { return g_pred; }

cudaError_t gemm_make_operand_map(CUtensorMap* out, const GemmOperand& op, DType dt,
                                  int rows_extent, int K, int batch, int rows_tile) {
  return make_map(out, op, dt, rows_extent, K, batch, rows_tile);
}

static int device_sms() {
  static const int sms = [] {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
      (void)cudaGetLastError();
      return 132;
    }
    return n;
  }();
  return sms;
}

int gemm_pick_bn(int N, EpiKind kind, int M, int z) {
  if (kind != EpiKind::GENERIC) return N <= 64 ? 64 : 128;
  // Largest tile that still yields ~a wave of CTAs; tiny problems take the narrowest tile so
  // the fixed per-CTA latency (setup + first TMA + epilogue) is spread over more SMs.
  const int mt = (M + kBM - 1) / kBM;
  const int cand[2] = {128, 64};
  for (int i = 0; i < 2; ++i) {
    const int bn = cand[i];
    if (bn > 64 && N <= bn / 2) continue;
    const long long ctas = static_cast<long long>((N + bn - 1) / bn) * mt * (z < 1 ? 1 : z);
    if (ctas * 10 >= device_sms() * 9 || bn == 64) return bn;   // >= ~0.9 of a wave
  }
  return 64;
}

cudaError_t gemm_make_b_map(const GemmProblem& p, CUtensorMap* out_host) {
  bind_context_once();
  // e4m3 GEMM launches run 64-wide tiles, so an e4m3 map defaults to the 64-row box; an explicit
  // force_bn (e.g. the 128-row box of the validation chain, mlp_val_sm100.cu) is kept
  const int BN = p.force_bn ? p.force_bn
                 : (p.ab_dtype == DType::FP8_E4M3 ? 64 : gemm_pick_bn(p.N, p.epi.kind, p.M, p.batch));
  return make_map(out_host, p.b, p.ab_dtype, p.N, p.K, p.batch, BN);
}

cudaError_t gemm_sm100(const GemmProblem& p, cudaStream_t stream) {
  bind_context_once();
  if (p.M <= 0 || p.N <= 0 || p.K <= 0 || p.batch <= 0) return cudaErrorInvalidValue;
  const bool fp8 = p.ab_dtype == DType::FP8_E4M3;
  if (p.ab_dtype == DType::F32) return cudaErrorInvalidValue;
  int BN = p.force_bn ? p.force_bn
                      : gemm_pick_bn(p.N, p.epi.kind, p.M,
                                     p.batch * (p.epi.split_k < 1 ? 1 : p.epi.split_k));
  if (BN != 64 && BN != 128) return cudaErrorInvalidValue;
  // e4m3 operands: K-major only and 64-wide tiles (room for the f16 copies, see kFp8Stages).
  // Decided before the row-wise check below: a row-wise epilogue needs the whole row in one tile,
  // and pre-built B maps (b_maps_dev) must have been encoded with the 64-row box.
  if (fp8 && (p.a.mn_major || p.b.mn_major)) return cudaErrorNotSupported;
  if (fp8 && p.b_maps_dev != nullptr && BN != 64) return cudaErrorNotSupported;
  if (fp8) BN = 64;
  if (p.epi.kind != EpiKind::GENERIC && (p.N > 128 || BN < p.N))
    return fp8 ? cudaErrorNotSupported : cudaErrorInvalidValue;
  // Split-K adds fp32 partial sums into d with atomics.  Bias (split 0 only) and column sums are
  // linear in the partial sums; an activation, its pre-activation copy or an activation-backward
  // mask applied to a partial sum is not, so those combinations are refused.
  if (p.epi.split_k > 1 &&
      (p.epi.kind != EpiKind::GENERIC || p.epi.d_dtype != DType::F32 || p.epi.act != Act::NONE ||
       p.epi.aux_out != nullptr || p.epi.act_bwd != 0))
    return cudaErrorInvalidValue;
  // accumulate (d += result) exists for fp32 d only; every other store overwrites d
  if (p.epi.accumulate && (p.epi.kind != EpiKind::GENERIC || p.epi.d_dtype != DType::F32))
    return cudaErrorInvalidValue;
  // the cross-entropy epilogue writes whole dlogits rows of ldd >= N columns
  if (p.epi.kind == EpiKind::XENT && p.epi.d != nullptr && p.epi.ldd < p.N)
    return cudaErrorInvalidValue;
  const int block_k = fp8 ? 128 : 64;
  const ConvView& cv = p.conv;
  // Low-rank K tail: one extra bf16 K block through the generic epilogue of a plain (batch 1,
  // single-split, overwriting) GEMM.  K2 a multiple of 8 keeps every tail row pitch 16-byte aligned.
  const bool tail = p.K2 != 0;
  if (tail) {
    if (p.K2 < 8 || p.K2 > 64 || p.K2 % 8 != 0 || p.a2.ptr == nullptr || p.b2.ptr == nullptr)
      return cudaErrorInvalidValue;
    if (fp8 || p.batch != 1 || p.epi.split_k > 1 || p.epi.accumulate || cv.mode != 0 ||
        p.b_maps_dev != nullptr || p.dyn != nullptr || p.epi.kind != EpiKind::GENERIC ||
        p.a2.mn_major != p.a.mn_major || p.b2.mn_major != p.b.mn_major)
      return cudaErrorNotSupported;
  }

  CUtensorMap ta, tb, tc, ta2, tb2;
  std::memset(&tc, 0, sizeof(tc));
  cudaError_t e = cudaSuccess;
  const int taps = cv.KH * cv.KW;
  if (cv.mode != 0) {
    if (fp8 || p.batch != 1 || p.b_maps_dev || p.dyn || p.epi.kind != EpiKind::GENERIC)
      return cudaErrorInvalidValue;
    if (cv.mode == 1) {
      // rows = pixels of the (OH, OW) grid; K = taps x C
      if (p.a.mn_major || p.K != taps * cv.C || p.M != cv.N * cv.OH * cv.OW) return cudaErrorInvalidValue;
      if (cv.flip && (cv.stride != 1 || !p.b.mn_major || p.N % 64 != 0)) return cudaErrorInvalidValue;
      if (!cv.flip && p.b.mn_major) return cudaErrorInvalidValue;
      if (cv.flip && BN > p.N) BN = (p.N % 128 == 0) ? 128 : 64;
      if (cv.flip && p.N % BN != 0) BN = 64;
      e = make_conv_map(&tc, cv, kBM);
      if (e != cudaSuccess) return e;
      std::memset(&ta, 0, sizeof(ta));
      e = cv.flip ? make_map(&tb, p.b, p.ab_dtype, taps * p.N, cv.C, 1, BN)
                  : make_map(&tb, p.b, p.ab_dtype, p.N, p.K, 1, BN);
      if (e != cudaSuccess) return e;
    } else {
      // D = dW [Cout][taps x C]; reduction over the pixels
      if (!p.a.mn_major || p.N != taps * cv.C || p.K != cv.N * cv.OH * cv.OW) return cudaErrorInvalidValue;
      BN = (cv.C % 128 == 0 && BN >= 128) ? 128 : 64;
      e = make_conv_map(&tc, cv, 64);
      if (e != cudaSuccess) return e;
      e = make_map(&ta, p.a, p.ab_dtype, p.M, p.K, 1, kBM);
      if (e != cudaSuccess) return e;
      std::memset(&tb, 0, sizeof(tb));
    }
  } else {
    e = make_map(&ta, p.a, p.ab_dtype, p.M, p.K, p.batch, kBM);
    if (e != cudaSuccess) return e;
    if (p.b_maps_dev == nullptr) {
      e = make_map(&tb, p.b, p.ab_dtype, p.N, p.K, p.batch, BN);
      if (e != cudaSuccess) return e;
    } else {
      std::memset(&tb, 0, sizeof(tb));
    }
    if (tail) {
      e = make_map(&ta2, p.a2, p.ab_dtype, p.M, p.K2, 1, kBM);
      if (e != cudaSuccess) return e;
      e = make_map(&tb2, p.b2, p.ab_dtype, p.N, p.K2, 1, BN);
      if (e != cudaSuccess) return e;
    }
  }

  KParams kp{};
  kp.M = p.M; kp.N = p.N; kp.K = p.K; kp.batch = p.batch;
  kp.is_fp8 = fp8 ? 1 : 0;
  kp.a_mn = p.a.mn_major ? 1 : 0;
  kp.b_mn = p.b.mn_major ? 1 : 0;
  kp.a_batched = (p.a.batch_stride != 0 && p.batch > 1) ? 1 : 0;
  kp.b_batched = (p.b.batch_stride != 0 && p.batch > 1) ? 1 : 0;
  kp.k_blocks = (p.K + block_k - 1) / block_k;
  kp.split_k = p.epi.split_k < 1 ? 1 : p.epi.split_k;
  if (kp.split_k > kp.k_blocks) kp.split_k = kp.k_blocks;
  kp.b_maps_dev = p.b_maps_dev;
  kp.dyn = p.dyn;
  kp.pred = current_predicate();
  kp.dbg_times = g_dbg_times;
  kp.d = p.epi.d;
  kp.d_dtype = static_cast<int>(p.epi.d_dtype);
  kp.ldd = p.epi.ldd;
  kp.d_batch_stride = p.epi.d_batch_stride;
  kp.alpha = p.epi.alpha;
  kp.bias = p.epi.bias;
  kp.bias_ptrs = p.epi.bias_ptrs;
  kp.act = static_cast<int>(p.epi.act);
  kp.aux_out = p.epi.aux_out;
  kp.aux_in = p.epi.aux_in;
  kp.act_bwd = p.epi.act_bwd;
  kp.colsum = p.epi.colsum;
  // split-K always adds into d, also when the clamp above leaves a single split
  kp.accumulate = (p.epi.accumulate || p.epi.split_k > 1) ? 1 : 0;
  kp.labels = p.epi.labels;
  kp.labels_batch_stride = p.epi.labels_batch_stride;
  kp.grad_scale = p.epi.grad_scale;
  kp.loss_sum = p.epi.loss_sum;
  kp.correct = p.epi.correct;
  {
    // vector (16 B fp32 / 8 B bf16) global access needs 4-element aligned rows everywhere
    auto al = [](const void* q, int bytes) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) % bytes) == 0; };
    const int eb = p.epi.d_dtype == DType::F32 ? 16 : (p.epi.d_dtype == DType::BF16 ? 8 : 4);
    kp.vec_ok = (p.epi.ldd % 4 == 0) && (p.epi.d_batch_stride % 4 == 0) && al(p.epi.d, eb) &&
                al(p.epi.aux_out, 8) && al(p.epi.aux_in, 8);
  }
  // Canonical SWIZZLE_128B descriptors.
  //  K-major : rows of 128 B; 8-row groups every 1024 B (SBO); LBO unused (1 unit).
  //            one MMA K-step = 32 B inside the swizzle span.
  //  MN-major: each TMA box is [block_k K-rows][128 B of MN]; 8-row K groups every 1024 B
  //            (SBO); the next 128-B MN chunk is the next box, block_k*128 B away (LBO);
  //            one MMA K-step = (32 / es) K-rows = 32/es * 128 B.
  const uint32_t mn_kstep = (fp8 ? 32u : 16u) * 128u;
  kp.lbo_a = p.dbg_lbo_a ? p.dbg_lbo_a : (p.a.mn_major ? static_cast<uint32_t>(block_k) * 128u : 16u);
  kp.sbo_a = p.dbg_sbo_a ? p.dbg_sbo_a : 1024u;
  kp.lbo_b = p.dbg_lbo_b ? p.dbg_lbo_b : (p.b.mn_major ? static_cast<uint32_t>(block_k) * 128u : 16u);
  kp.sbo_b = p.dbg_sbo_b ? p.dbg_sbo_b : 1024u;
  kp.kstep_a = p.a.mn_major ? mn_kstep : 32u;
  kp.kstep_b = p.b.mn_major ? mn_kstep : 32u;
  kp.cv_mode = cv.mode; kp.cv_flip = cv.flip;
  kp.cv_cb = cv.C / 64; kp.cv_kw = cv.KW; kp.cv_pad = cv.pad; kp.cv_stride = cv.stride;
  kp.cv_oh = cv.OH; kp.cv_ow = cv.OW; kp.cv_c = cv.C;
  if (cv.mode == 2) kp.b_mn = 1;  // shifted activation boxes are [pixels][channels]: MN-major B
  if (cv.mode == 2) { kp.lbo_b = 64u * 128u; kp.kstep_b = mn_kstep; }

  dim3 grid((p.N + BN - 1) / BN, (p.M + kBM - 1) / kBM, p.batch * kp.split_k);
  {
    // Ring depth: the full ring (BFLC_GEMM_STAGES overrides it for experiments).
    const int full = BN == 128 ? 4 : 6;
    static const int force = [] { const char* e = std::getenv("BFLC_GEMM_STAGES"); return e ? std::atoi(e) : 0; }();
    kp.stages = full;
    if (force >= 2 && force <= full) kp.stages = force;
    if (fp8) kp.stages = kFp8Stages;
  }
  if (tail) {
    if (BN == 64) return launch_tail<64>(ta, tb, tc, kp, ta2, tb2, grid, stream);
    return launch_tail<128>(ta, tb, tc, kp, ta2, tb2, grid, stream);
  }
#define BFLC_LAUNCH(BN_, EPI_) return launch<BN_, EPI_>(ta, tb, tc, kp, grid, stream)
  const int epi = static_cast<int>(p.epi.kind);
  if (epi == 0) {
    if (BN == 64) BFLC_LAUNCH(64, 0);
    BFLC_LAUNCH(128, 0);
  } else if (epi == 1) {
    if (BN == 64) BFLC_LAUNCH(64, 1);
    BFLC_LAUNCH(128, 1);
  } else {
    if (BN == 64) BFLC_LAUNCH(64, 2);
    BFLC_LAUNCH(128, 2);
  }
#undef BFLC_LAUNCH
}

// Implicit-GEMM weight gradient of a convolution by K groups (conv mode 2, EPI 3): the pixels of x / dy split
// into `groups` equal runs of whole examples, group g one CTA layer (grid z) reducing its own K blocks.
// sq != nullptr: per-example squared norms, sq[tile * groups + g] = ||tile of dW_g||^2 over the
// ceil(Cout / 128) x (taps C / 64) tiles (conv_dw_norm_tiles); else d [groups][Cout][taps C] fp32 gets each
// group's dW_g with plain stores (a deterministic split-K's slices).  Refused before launch: fp8, a split-K,
// accumulate, bias, activation or column sums, and groups whose pixels the 64-pixel boxes do not tile.
int conv_dw_norm_tiles(int Cout, int K) { return ((Cout + kBM - 1) / kBM) * (K / 64); }

cudaError_t conv_dw_groups(const GemmProblem& p, int groups, float* sq, cudaStream_t stream) {
  bind_context_once();
  const ConvView& cv = p.conv;
  const long long pixels = static_cast<long long>(cv.N) * cv.OH * cv.OW;
  if (cv.mode != 2 || groups < 1 || p.batch != 1 || p.ab_dtype != DType::BF16 || p.epi.split_k > 1 ||
      p.epi.accumulate || p.epi.bias != nullptr || p.epi.act != Act::NONE || p.epi.aux_out != nullptr ||
      p.epi.aux_in != nullptr || p.epi.act_bwd != 0 || p.epi.colsum != nullptr ||
      p.epi.kind != EpiKind::GENERIC || p.b_maps_dev != nullptr || p.dyn != nullptr || p.K2 != 0)
    return cudaErrorInvalidValue;
  if (cv.N % groups != 0 || (pixels / groups) % 64 != 0 || cv.C % 64 != 0) return cudaErrorInvalidValue;
  if (!p.a.mn_major || p.N != cv.KH * cv.KW * cv.C || p.K != pixels || p.M < 1) return cudaErrorInvalidValue;
  if (sq == nullptr && (p.epi.d == nullptr || p.epi.d_dtype != DType::F32 ||
                        p.epi.d_batch_stride < static_cast<int64_t>(p.M) * p.epi.ldd || p.epi.ldd < p.N))
    return cudaErrorInvalidValue;
  constexpr int BN = 64;
  CUtensorMap ta, tb, tc;
  std::memset(&tb, 0, sizeof(tb));
  cudaError_t e = make_conv_map(&tc, cv, 64);
  if (e != cudaSuccess) return e;
  e = make_map(&ta, p.a, p.ab_dtype, p.M, p.K, 1, kBM);
  if (e != cudaSuccess) return e;
  KParams kp{};
  kp.M = p.M; kp.N = p.N; kp.K = p.K; kp.batch = groups;
  kp.a_mn = 1; kp.b_mn = 1;
  kp.k_blocks = static_cast<int>(pixels / 64);
  kp.split_k = 1;
  kp.group_kb = static_cast<int>(pixels / groups / 64);
  kp.pe_sq = sq;
  kp.pred = current_predicate();
  kp.d = sq == nullptr ? p.epi.d : nullptr;
  kp.d_dtype = 0;
  kp.ldd = p.epi.ldd;
  kp.d_batch_stride = p.epi.d_batch_stride;
  kp.alpha = 1.f;
  kp.vec_ok = (p.epi.ldd % 4 == 0) && (p.epi.d_batch_stride % 4 == 0) &&
              (reinterpret_cast<uintptr_t>(p.epi.d) % 16 == 0);
  const uint32_t mn_kstep = 16u * 128u;
  kp.lbo_a = 64u * 128u; kp.sbo_a = 1024u; kp.kstep_a = mn_kstep;
  kp.lbo_b = 64u * 128u; kp.sbo_b = 1024u; kp.kstep_b = mn_kstep;
  kp.cv_mode = 2; kp.cv_flip = 0;
  kp.cv_cb = cv.C / 64; kp.cv_kw = cv.KW; kp.cv_pad = cv.pad; kp.cv_stride = cv.stride;
  kp.cv_oh = cv.OH; kp.cv_ow = cv.OW; kp.cv_c = cv.C;
  kp.stages = SmemLayout<BN>::kStages;
  const dim3 grid(p.N / BN, (p.M + kBM - 1) / kBM, groups);
  return launch<BN, 3>(ta, tb, tc, kp, grid, stream);
}

}  // namespace bflc
