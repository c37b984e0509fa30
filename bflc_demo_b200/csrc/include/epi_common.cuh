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

#include "bflc_kernels.h"
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
// UE8M0 exponent byte for a group whose largest magnitude is amax: 2^(e-127) >= amax / 448.
// Clamped to [kMx8MinScale, 254]: from e = 3 up, every e4m3 value times 2^(e-127) is a bf16 value
// (mx8_dq1), so the tensor cores can run the block-scaled product as a bf16 GEMM.  Only groups with
// amax < 448 * 2^-125 (~1.3e-35) ever needed a smaller byte.
constexpr int kMx8MinScale = 3;
__device__ __forceinline__ int mx8_scale_byte(float amax) {
  if (!(amax > 0.f)) return 127;
  const uint32_t b = __float_as_uint(amax * (1.f / 448.f));
  int e = static_cast<int>((b >> 23) & 0xFF) + ((b & 0x7FFFFF) ? 1 : 0);
  return max(kMx8MinScale, min(254, e));
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

// e4m3 value q (as the f16 bits h the hardware converts it to, exactly) times 2^(e-127) -> bf16
// bits, by integer arithmetic: no float multiply, so no flush-to-zero under fast-math.  Exact for
// 3 <= e <= 246: q's lowest set bit is >= 2^-9 and q has at most 4 significant bits, so
// q * 2^(e-127) is a multiple of 2^-133 (the bf16 subnormal step) and below the bf16 maximum.
// Results under 2^-126 become bf16 subnormals (only for e <= 9).  DESIGN.md §3.
__device__ __forceinline__ uint32_t mx8_dq1(uint32_t h, int e) {
  const uint32_t mag = h & 0x7FFFu;
  const int x = static_cast<int>(mag >> 10) + e - 15;    // biased bf16 exponent of the product
  const uint32_t m7 = (mag >> 3) & 0x7Fu;                // e4m3 has 3 mantissa bits: nothing is lost
  const uint32_t b = mag == 0u ? 0u : x > 0 ? (static_cast<uint32_t>(x) << 7) | m7 : (0x80u | m7) >> (1 - x);
  return (h & 0x8000u) | b;
}
// mx8_dq1 on both halves of a packed pair of e4m3-derived f16 bits, for scale bytes e >= 10.  Every
// nonzero e4m3 value (NaN and the saturation band included) is an f16 with biased exponent >= 6 and
// a zero low 3 mantissa bits, so mx8_dq1's x is positive and its result is
// sign | (mag >> 3) + ((e - 15) << 7); a zero magnitude keeps only the sign.  Per half,
// t = mag >> 3 < 2^12 (the mask drops the sign and the bits the shift moves across the halves), bit
// 12 of t + 0xFFF flags t != 0, and t + ((e - 15) << 7) < 2^16, so no carry crosses a half.  Bit for
// bit mx8_dq1 over every e4m3 value and every such e, in about a third of its integer work.
__device__ __forceinline__ uint32_t mx8_dq2_normal(uint32_t h2, int e) {
  const uint32_t t = (h2 >> 3) & 0x0FFF0FFFu;
  const uint32_t nz = ((t + 0x0FFF0FFFu) >> 12) & 0x00010001u;
  return (t + nz * (static_cast<uint32_t>(e - 15) << 7)) | (h2 & 0x80008000u);
}
// scale bytes 3..9 (groups with amax below ~1.2e-33), whose products may be bf16 subnormals.  Not
// inlined: a second inlined copy at every call site raised the persistent trainer's register spills
static __device__ __noinline__ uint2 mx8_dq4_slow(uint32_t w, int e) {
  const __half2_raw lo = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w & 0xFFFFu), __NV_E4M3);
  const __half2_raw hi = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w >> 16), __NV_E4M3);
  return make_uint2(mx8_dq1(lo.x, e) | (mx8_dq1(lo.y, e) << 16), mx8_dq1(hi.x, e) | (mx8_dq1(hi.y, e) << 16));
}
// four e4m3 bytes (w, lowest byte first) with scale byte e -> four bf16 (two packed pairs)
__device__ __forceinline__ uint2 mx8_dq4(uint32_t w, int e) {
  if (e < 10) return mx8_dq4_slow(w, e);
  const __half2_raw lo = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w & 0xFFFFu), __NV_E4M3);
  const __half2_raw hi = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w >> 16), __NV_E4M3);
  return make_uint2(mx8_dq2_normal(lo.x | (static_cast<uint32_t>(lo.y) << 16), e),
                    mx8_dq2_normal(hi.x | (static_cast<uint32_t>(hi.y) << 16), e));
}
// eight e4m3 words (32 elements of one K-group) -> 64 bytes of bf16 at dst (16-byte aligned)
__device__ __forceinline__ void mx8_dq32_store(const uint32_t (&w)[8], int e, __nv_bfloat16* dst, int n = 32) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (i * 8 >= n) break;
    const uint2 a = mx8_dq4(w[2 * i], e), b = mx8_dq4(w[2 * i + 1], e);
    reinterpret_cast<uint4*>(dst)[i] = make_uint4(a.x, a.y, b.x, b.y);
  }
}

// Unpacking a candidate's MXFP8 blob (Mx8MlpLayout) for validation: the e4m3 weights become the
// exactly dequantised bf16 matrices of a flat parameter slot (W1 at w1_off, W2 at w2_off, n_classes
// rows), the fp32 biases are copied into the local blob slot.  The work is a list of 16-byte
// units -- W1 e4m3 chunks, W2 e4m3 chunks, bias chunks -- so that callers can split it between
// threads / CTAs; every source byte is read once, with relaxed system-scope loads (the blob may
// be in a peer's HBM, rewritten every second round).
__host__ __device__ __forceinline__ long long mx8_unpack_units(const Mx8Unpack& u) {
  return static_cast<long long>(u.hidden) * (u.in_dim / 16) + static_cast<long long>(u.n_classes) * (u.hidden / 16) +
         (u.hidden + 64) / 4;
}
__device__ __forceinline__ uint32_t ld_peer_u32(const void* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ int ld_peer_scale(const uint8_t* chunks, long long idx) {
  return static_cast<int>((ld_peer_u32(chunks + (idx & ~3LL)) >> (8 * (idx & 3))) & 0xFFu);
}
__device__ __forceinline__ void mx8_unpack_unit(const Mx8Unpack& u, const uint8_t* src, __nv_bfloat16* dst,
                                                uint8_t* dst_blob, long long i) {
  const long long n1 = static_cast<long long>(u.hidden) * (u.in_dim / 16);
  const long long n2 = static_cast<long long>(u.n_classes) * (u.hidden / 16);
  if (i >= n1 + n2) {   // fp32 biases b1 | b2, 16 bytes at a time
    const long long o = u.b1 + 16 * (i - n1 - n2);
    *reinterpret_cast<float4*>(dst_blob + o) = ptx::ld_peer_f4(reinterpret_cast<const float4*>(src + o));
    return;
  }
  const bool l1 = i < n1;
  const long long j = l1 ? i : i - n1;
  const int ld = l1 ? u.in_dim : u.hidden, per = ld / 16;
  const int row = static_cast<int>(j / per), c = static_cast<int>(j % per) * 16;
  const long long off = static_cast<long long>(row) * ld + c;
  const float4 q4 = ptx::ld_peer_f4(reinterpret_cast<const float4*>(src + (l1 ? u.w1q : u.w2q) + off));
  const int e = ld_peer_scale(src + (l1 ? u.w1sf : u.w2sf), mx8_sf_index(row, c >> 5, l1 ? u.kb1 : u.kb2));
  const uint32_t w[4] = {__float_as_uint(q4.x), __float_as_uint(q4.y), __float_as_uint(q4.z), __float_as_uint(q4.w)};
  const uint2 a = mx8_dq4(w[0], e), b = mx8_dq4(w[1], e), c2 = mx8_dq4(w[2], e), d = mx8_dq4(w[3], e);
  uint4* o = reinterpret_cast<uint4*>(dst + (l1 ? u.w1_off : u.w2_off) + off);
  o[0] = make_uint4(a.x, a.y, b.x, b.y);
  o[1] = make_uint4(c2.x, c2.y, d.x, d.y);
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
