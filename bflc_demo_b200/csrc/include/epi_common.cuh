// Device helpers shared by the tensor-core kernels of the library (gemm_sm100.cu,
// gemm_mx8_sm100.cu, mlp_round_sm100.cu, mlp_val_sm100.cu): the per-warp [32][36] fp32 staging
// tile that turns "one accumulator row per thread" into stores that cover 4 whole rows x 128 B per
// instruction, 128-byte-swizzle addressing, and the block-scaled-fp8 (MXFP8) primitives -- the
// scale-chunk layout, its bulk copy and the quantiser arithmetic.
//
// No reference counterpart: the reference (iammcy/BFLC-demo) has no GPU code (SURVEY.md 2.7).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp8.h>

#include <cstdint>

#include "sm100_ptx.cuh"

namespace bflc {
namespace epi {

constexpr int kStgLd = 36;  // floats per staged row: 16-byte aligned, conflict-free both ways
constexpr int kStgWarpFloats = 32 * kStgLd;
constexpr int kStgBytes = 4 * kStgWarpFloats * 4;  // four epilogue warps

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ void stage_put(float* stg, int lane, const float (&v)[32]) {
  float4* rowp = reinterpret_cast<float4*>(stg + lane * kStgLd);
#pragma unroll
  for (int j = 0; j < 8; ++j) rowp[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
}
__device__ __forceinline__ void stage_get(const float* stg, int lane, float (&v)[32]) {
  const float4* rowp = reinterpret_cast<const float4*>(stg + lane * kStgLd);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 t = rowp[j];
    v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
  }
}
// sum of column `lane` over the first rmax rows of a staged 32 x 32 sub-tile: all 32 loads are
// independent and issued back to back (a rolled `tot += stg[...]` loop serialised ~25-cycle smem
// latencies: 0.4 us per sub-tile, 3+ us per dh tile -- measured with the in-kernel stamps)
__device__ __forceinline__ float col_sum32(const float* stg, int lane, int rmax) {
  float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int rr = 0; rr < 32; ++rr) t[rr & 3] += rr < rmax ? stg[rr * kStgLd + lane] : 0.f;
  return (t[0] + t[1]) + (t[2] + t[3]);
}
// 16-byte chunk `chunk` of row r of a 128-byte-swizzled K-major operand tile
__device__ __forceinline__ void st_sw128(uint8_t* tile, int r, int chunk, uint4 v) {
  *reinterpret_cast<uint4*>(tile + r * 128 + ((chunk ^ (r & 7)) << 4)) = v;
}
__device__ __forceinline__ uint4 ld_sw128(const uint8_t* tile, int r, int chunk) {
  return *reinterpret_cast<const uint4*>(tile + r * 128 + ((chunk ^ (r & 7)) << 4));
}

// ---------------------------------------------------------------------------------- MXFP8
// OCP MXFP8: e4m3 elements, one UE8M0 scale per 32 consecutive K-elements.  Scale factors live
// in global memory in the order the tensor core consumes them: per (128-row block, 128-K block)
// one 512-byte chunk whose byte [r % 32][r / 32][k / 32] scales row r, K-group k; chunks are
// stored [row_block][k_block].  One `cp.async.bulk` moves a chunk to smem, where the MMA warpgroup
// reads each fragment row's / column's byte (wg::mx_accumulate).
constexpr int kSfChunk = 512;

__host__ __device__ constexpr int mx8_sf_off(int r128, int g4) {
  return (r128 & 31) * 16 + (r128 >> 5) * 4 + g4;
}
// byte offset of the scale of (row, K-group g) inside a chunk array with n_kb K-blocks per row block
__host__ __device__ constexpr long long mx8_sf_index(int row, int g, int n_kb) {
  return (static_cast<long long>(row >> 7) * n_kb + (g >> 2)) * kSfChunk + mx8_sf_off(row & 127, g & 3);
}
// UE8M0 exponent byte for a group whose largest magnitude is amax: 2^(e-127) >= amax / 448
__device__ __forceinline__ int mx8_scale_byte(float amax) {
  if (!(amax > 0.f)) return 127;
  const uint32_t b = __float_as_uint(amax * (1.f / 448.f));
  int e = static_cast<int>((b >> 23) & 0xFF) + ((b & 0x7FFFFF) ? 1 : 0);
  return max(1, min(254, e));
}
__device__ __forceinline__ float mx8_inv_scale(int e) {   // 2^(127 - e)
  return __uint_as_float(static_cast<uint32_t>(254 - e) << 23);
}
__device__ __forceinline__ uint32_t mx8_pack4(float a, float b, float c, float d) {
  const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
  const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
  return lo | (hi << 16);
}
// quantise one 32-element K-group held by a single thread: returns the scale byte, w[8] = 32 e4m3
__device__ __forceinline__ int mx8_quant32(const float (&v)[32], uint32_t (&w)[8]) {
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) amax = fmaxf(amax, fabsf(v[i]));
  const int e = mx8_scale_byte(amax);
  const float inv = mx8_inv_scale(e);
#pragma unroll
  for (int i = 0; i < 8; ++i)
    w[i] = mx8_pack4(v[4 * i] * inv, v[4 * i + 1] * inv, v[4 * i + 2] * inv, v[4 * i + 3] * inv);
  return e;
}

__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(ptx::smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes),
        "r"(ptx::smem_u32(bar))
      : "memory");
}
}  // namespace epi
}  // namespace bflc
