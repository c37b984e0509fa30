// Bandwidth-bound helpers: dtype casts / fp8 quantisation, and the fused flat-buffer
// optimizers.  Every kernel is vectorised to 16-byte accesses and sized as a grid-stride
// loop over 132 SMs x 8 CTAs.
//
// Optimizer parity: the reference trains with tf.train.GradientDescentOptimizer(0.001)
// and keeps Adam as a commented-out alternative (python-sdk/main.py:126-130); both are
// first-class here.  The update also refreshes the bf16 "shadow" weights the tensor-core
// GEMMs read, so no separate cast pass ever touches the parameters.
#include <cuda_bf16.h>
#include <cuda_fp8.h>

#include "bflc_kernels.h"
#include "epi_common.cuh"
#include "launch.cuh"
#include "sm100_ptx.cuh"

namespace bflc {

namespace {

constexpr int kBlock = 256;
inline int grid_for(int64_t n_vec) {
  int64_t g = (n_vec + kBlock - 1) / kBlock;
  const int64_t cap = 132 * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<int>(g);
}

using epi::pack_bf16x2;

__global__ void k_cast_f32_bf16(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                int64_t n) {
  const int64_t nv = n / 8;
  const int64_t tid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = tid; i < nv; i += stride) {
    const float4 a = reinterpret_cast<const float4*>(src)[2 * i];
    const float4 b = reinterpret_cast<const float4*>(src)[2 * i + 1];
    uint4 o;
    o.x = pack_bf16x2(a.x, a.y); o.y = pack_bf16x2(a.z, a.w);
    o.z = pack_bf16x2(b.x, b.y); o.w = pack_bf16x2(b.z, b.w);
    reinterpret_cast<uint4*>(dst)[i] = o;
  }
  for (int64_t i = nv * 8 + tid; i < n; i += stride) dst[i] = __float2bfloat16(src[i]);
}

__global__ void k_cast_bf16_f32(const __nv_bfloat16* __restrict__ src, float* __restrict__ dst,
                                int64_t n) {
  const int64_t tid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = tid; i < n; i += stride) dst[i] = __bfloat162float(src[i]);
}

__global__ void k_cast_u8_bf16(const uint8_t* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                               int64_t n, float scale, const int* pred) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  if (pred != nullptr && *pred == 0) return;
  const int64_t nv = n / 16;
  const int64_t tid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = tid; i < nv; i += stride) {
    const uint4 in = reinterpret_cast<const uint4*>(src)[i];
    const uint32_t w[4] = {in.x, in.y, in.z, in.w};
    uint32_t o[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      o[2 * k] = pack_bf16x2((w[k] & 0xff) * scale, ((w[k] >> 8) & 0xff) * scale);
      o[2 * k + 1] = pack_bf16x2(((w[k] >> 16) & 0xff) * scale, (w[k] >> 24) * scale);
    }
    reinterpret_cast<uint4*>(dst)[2 * i] = make_uint4(o[0], o[1], o[2], o[3]);
    reinterpret_cast<uint4*>(dst)[2 * i + 1] = make_uint4(o[4], o[5], o[6], o[7]);
  }
  for (int64_t i = nv * 16 + tid; i < n; i += stride) dst[i] = __float2bfloat16(src[i] * scale);
}

__global__ void k_quant_fp8(const __nv_bfloat16* __restrict__ src, uint8_t* __restrict__ dst,
                            int64_t n, float inv_scale) {
  const int64_t tid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const int64_t nv = n / 8;
  for (int64_t i = tid; i < nv; i += stride) {
    const uint4 in = reinterpret_cast<const uint4*>(src)[i];
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&in);
    uint8_t o[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = __bfloat1622float2(h[k]);
      o[2 * k] = __nv_cvt_float_to_fp8(f.x * inv_scale, __NV_SATFINITE, __NV_E4M3);
      o[2 * k + 1] = __nv_cvt_float_to_fp8(f.y * inv_scale, __NV_SATFINITE, __NV_E4M3);
    }
    reinterpret_cast<uint2*>(dst)[i] = *reinterpret_cast<uint2*>(o);
  }
  for (int64_t i = nv * 8 + tid; i < n; i += stride)
    dst[i] = __nv_cvt_float_to_fp8(__bfloat162float(src[i]) * inv_scale, __NV_SATFINITE, __NV_E4M3);
}

__global__ void k_amax_bf16(const __nv_bfloat16* __restrict__ src, int64_t n, float* out) {
  const int64_t tid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  float m = 0.f;
  for (int64_t i = tid; i < n; i += stride) m = fmaxf(m, fabsf(__bfloat162float(src[i])));
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  // non-negative floats order like their bit patterns
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(out), __float_as_int(m));
}

__global__ void k_fill(float* dst, int64_t n, float v) {
  const int64_t tid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = tid; i < n; i += stride) dst[i] = v;
}

__global__ void k_add_bf16(const __nv_bfloat16* a, const __nv_bfloat16* b, __nv_bfloat16* o,
                           int64_t n) {
  const int64_t tid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const int64_t nv = n / 8;
  for (int64_t i = tid; i < nv; i += stride) {
    const uint4 x = reinterpret_cast<const uint4*>(a)[i];
    const uint4 y = reinterpret_cast<const uint4*>(b)[i];
    const __nv_bfloat162* hx = reinterpret_cast<const __nv_bfloat162*>(&x);
    const __nv_bfloat162* hy = reinterpret_cast<const __nv_bfloat162*>(&y);
    uint4 r;
    uint32_t* ro = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 fx = __bfloat1622float2(hx[k]);
      const float2 fy = __bfloat1622float2(hy[k]);
      ro[k] = pack_bf16x2(fx.x + fy.x, fx.y + fy.y);
    }
    reinterpret_cast<uint4*>(o)[i] = r;
  }
  for (int64_t i = nv * 8 + tid; i < n; i += stride)
    o[i] = __float2bfloat16(__bfloat162float(a[i]) + __bfloat162float(b[i]));
}

// ------------------------------------------------------------------ optimizers
// The recipe instantiations (kRecipe) take RecipeArgs; the others keep OptimArgs as it is, and with
// kRecipe false every recipe term below is compiled out.
template <bool kRecipe>
using OptimParams = typename std::conditional<kRecipe, RecipeArgs, OptimArgs>::type;

// lr factor f(s) of the HF get_{constant,linear,cosine}_schedule_with_warmup lambdas (s 0-based);
// double, so that the cosine is not the fast-math one
__device__ __forceinline__ float lr_factor(int schedule, int warmup, int total, int s) {
  if (s < warmup) return static_cast<float>(static_cast<double>(s) / static_cast<double>(warmup));
  if (schedule == kLrConstant) return 1.f;
  const double span = static_cast<double>(max(1, total - warmup));
  if (schedule == kLrLinear) return static_cast<float>(fmax(0.0, static_cast<double>(total - s) / span));
  return static_cast<float>(fmax(0.0, 0.5 * (1.0 + cospi(static_cast<double>(s - warmup) / span))));
}

// decoupled decay of 8-float block j: 0 when its no-decay bit is set
__device__ __forceinline__ float block_decay(const uint32_t* no_decay, int64_t j, float dec) {
  return no_decay != nullptr && ((__ldg(no_decay + (j >> 5)) >> (j & 31)) & 1u) ? 0.f : dec;
}

// One float of the recipe update.  The roundings are spelled out as intrinsics in the form the plain
// instantiations compile to (g = fma(wd, w, g); m = fma(b1, m, (1 - b1) g); v = fma(b2, v, g ((1 - b2) g));
// SGD w = fma(-lr, g, w)): left to contraction, nvcc fuses the other product of b1 m + (1 - b1) g in
// some loops, and the no-op recipe would drift from optim_step by an ulp.  w is decayed (keep =
// 1 - lr_t decay) after the coupled term has read it, as AdamW does.
template <bool kAdam>
__device__ __forceinline__ void recipe_update(float& w, float& m, float& v, float g_in, float keep, const RecipeArgs& a,
                                              float lr, float bc1, float bc2) {
  const float g = __fmaf_rn(a.weight_decay, w, g_in);
  w = __fmul_rn(w, keep);
  if (kAdam) {
    m = __fmaf_rn(a.beta1, m, __fmul_rn(1.f - a.beta1, g));
    v = __fmaf_rn(a.beta2, v, __fmul_rn(g, __fmul_rn(1.f - a.beta2, g)));
    w -= lr * (m / bc1) / (sqrtf(v / bc2) + a.eps);
  } else {
    w = __fmaf_rn(-lr, g, w);
  }
}

// FedProx: g' = fma(mu, w - w0, g), w the master before this step (before the decay), w0 the anchor.
// Callers test a.anchor first: without an anchor g stays exactly g (fma(0, d, -0) would be +0).
__device__ __forceinline__ float prox_grad(float g, float w, float w0, float mu) {
  return __fmaf_rn(mu, __fsub_rn(w, w0), g);
}

template <bool kAdam, bool kRecipe = false>
__global__ void k_optim(OptimParams<kRecipe> a) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  if (a.active != nullptr && *a.active == 0) return;
  const int64_t tid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  float bc1 = 1.f, bc2 = 1.f;
  if (kAdam) {
    const int t = (a.step_dev ? *a.step_dev : 0) + a.step;
    bc1 = 1.f - powf(a.beta1, static_cast<float>(t));
    bc2 = 1.f - powf(a.beta2, static_cast<float>(t));
  }
  // recipe: lr_t = lr f(t - 1), the clip coefficient (read after pdl_wait: grad_norm_f32 is the PDL
  // predecessor), decoupled decay lr_t * decay
  float lr = a.lr, coef = 1.f, dec = 0.f;
  if constexpr (kRecipe) {
    if (a.clip != nullptr) {
      coef = a.clip->coef;
      if (a.clip->nonfinite) {   // skipped step: weights and moments untouched, the gradient cleared
        if (a.zero_grad) {
          float* g = const_cast<float*>(a.grad);
          for (int64_t i = tid; i < a.n / 4; i += stride)
            reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int64_t i = a.n / 4 * 4 + tid; i < a.n; i += stride) g[i] = 0.f;
        }
        return;
      }
    }
    const int t = (a.step_dev ? *a.step_dev : 0) + a.step;
    lr = a.lr * lr_factor(a.schedule, a.warmup, a.total, t - 1);
    dec = lr * a.decay;
  }
  const int64_t nv = a.n / 4;
  __nv_bfloat16* sh = reinterpret_cast<__nv_bfloat16*>(a.shadow_bf16);
  for (int64_t i = tid; i < nv; i += stride) {
    float4 w = reinterpret_cast<float4*>(a.master)[i];
    const float4 g4 = reinterpret_cast<const float4*>(a.grad)[i];
    float wv[4] = {w.x, w.y, w.z, w.w};
    const float gv[4] = {g4.x, g4.y, g4.z, g4.w};
    float keep = 1.f;   // recipe: 1 - lr_t * decay of this float4's 8-float block
    float gq[4] = {gv[0], gv[1], gv[2], gv[3]};   // recipe: the gradient the update consumes
    if constexpr (kRecipe) {
      keep = 1.f - block_decay(a.no_decay, i >> 1, dec);
#pragma unroll
      for (int k = 0; k < 4; ++k) gq[k] = __fmul_rn(coef, gv[k]);
      if (a.anchor != nullptr) {
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(a.anchor) + i);
        gq[0] = prox_grad(gq[0], wv[0], w0.x, a.mu); gq[1] = prox_grad(gq[1], wv[1], w0.y, a.mu);
        gq[2] = prox_grad(gq[2], wv[2], w0.z, a.mu); gq[3] = prox_grad(gq[3], wv[3], w0.w, a.mu);
      }
    }
    if (kAdam) {
      float4 m4 = reinterpret_cast<float4*>(a.m)[i];
      float4 v4 = reinterpret_cast<float4*>(a.v)[i];
      float mv[4] = {m4.x, m4.y, m4.z, m4.w};
      float vv[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if constexpr (kRecipe) {
          recipe_update<true>(wv[k], mv[k], vv[k], gq[k], keep, a, lr, bc1, bc2);
        } else {
          const float g = gv[k] + a.weight_decay * wv[k];
          mv[k] = a.beta1 * mv[k] + (1.f - a.beta1) * g;
          vv[k] = a.beta2 * vv[k] + (1.f - a.beta2) * g * g;
          wv[k] -= a.lr * (mv[k] / bc1) / (sqrtf(vv[k] / bc2) + a.eps);
        }
      }
      reinterpret_cast<float4*>(a.m)[i] = make_float4(mv[0], mv[1], mv[2], mv[3]);
      reinterpret_cast<float4*>(a.v)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if constexpr (kRecipe) {
          float m_unused = 0.f, v_unused = 0.f;
          recipe_update<false>(wv[k], m_unused, v_unused, gq[k], keep, a, lr, bc1, bc2);
        } else {
          wv[k] -= a.lr * (gv[k] + a.weight_decay * wv[k]);
        }
      }
    }
    reinterpret_cast<float4*>(a.master)[i] = make_float4(wv[0], wv[1], wv[2], wv[3]);
    if (sh) {
      uint2 o;
      o.x = pack_bf16x2(wv[0], wv[1]);
      o.y = pack_bf16x2(wv[2], wv[3]);
      reinterpret_cast<uint2*>(sh)[i] = o;
    }
    if (a.zero_grad)
      reinterpret_cast<float4*>(const_cast<float*>(a.grad))[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int64_t i = nv * 4 + tid; i < a.n; i += stride) {
    float w = a.master[i];
    if constexpr (kRecipe) {
      float m = kAdam ? a.m[i] : 0.f, v = kAdam ? a.v[i] : 0.f;
      float g = __fmul_rn(coef, a.grad[i]);
      if (a.anchor != nullptr) g = prox_grad(g, w, __ldg(a.anchor + i), a.mu);
      recipe_update<kAdam>(w, m, v, g, 1.f - block_decay(a.no_decay, i >> 3, dec), a, lr, bc1, bc2);
      if (kAdam) { a.m[i] = m; a.v[i] = v; }
    } else {
      float g = a.grad[i] + a.weight_decay * w;
      if (kAdam) {
        const float m = a.beta1 * a.m[i] + (1.f - a.beta1) * g;
        const float v = a.beta2 * a.v[i] + (1.f - a.beta2) * g * g;
        a.m[i] = m; a.v[i] = v;
        w -= a.lr * (m / bc1) / (sqrtf(v / bc2) + a.eps);
      } else {
        w -= a.lr * g;
      }
    }
    a.master[i] = w;
    if (sh) sh[i] = __float2bfloat16(w);
    if (a.zero_grad) const_cast<float*>(a.grad)[i] = 0.f;
  }
}

// Global gradient norm for clipping.  Each thread sums the squares of its grid-stride share in fp64,
// in a fixed order; the CTA reduces with a fixed shuffle tree and writes one partial; the CTA that
// takes the last ticket sums the partials in index order and resets the ticket.  The grid depends
// only on n, so the result is bit-identical across calls and graph replays.  No float atomics.
struct NormArgs {
  const float* grad; int64_t n; GradNormState* st; double* partials; float* norm_out; float max_norm;
  int* skipped; const int* active;
};

__device__ __forceinline__ double block_sum(double x, double* red) {
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = x;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int w = 0; w < kBlock / 32; ++w) s += red[w];
  return s;
}

__global__ void __launch_bounds__(kBlock) k_grad_norm(NormArgs a) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  if (a.active != nullptr && *a.active == 0) return;
  __shared__ double red[kBlock / 32];
  __shared__ bool last;
  const int64_t tid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const int64_t nv = a.n / 4;
  double acc = 0.0;
  for (int64_t i = tid; i < nv; i += stride) {
    const float4 g = reinterpret_cast<const float4*>(a.grad)[i];
    acc = fma(static_cast<double>(g.x), static_cast<double>(g.x), acc);
    acc = fma(static_cast<double>(g.y), static_cast<double>(g.y), acc);
    acc = fma(static_cast<double>(g.z), static_cast<double>(g.z), acc);
    acc = fma(static_cast<double>(g.w), static_cast<double>(g.w), acc);
  }
  for (int64_t i = nv * 4 + tid; i < a.n; i += stride) acc = fma(static_cast<double>(a.grad[i]), static_cast<double>(a.grad[i]), acc);
  const double cta = block_sum(acc, red);
  if (threadIdx.x == 0) {
    a.partials[blockIdx.x] = cta;
    __threadfence();
    last = atomicAdd(&a.st->ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  double p = 0.0;
  for (int j = threadIdx.x; j < static_cast<int>(gridDim.x); j += kBlock) p += __ldcg(a.partials + j);
  __syncthreads();   // red[] is reused
  const double total = block_sum(p, red);
  if (threadIdx.x == 0) {
    const float norm = static_cast<float>(sqrt(total));
    const bool bad = !isfinite(norm);
    *a.norm_out = norm;
    a.st->coef = bad ? 1.f : fminf(1.f, __fdiv_rn(a.max_norm, norm + 1e-6f));
    a.st->nonfinite = bad ? 1 : 0;
    if (bad && a.skipped != nullptr) *a.skipped += 1;
    a.st->ticket = 0u;
  }
}

// ------------------------------------------------------------------ input preparation
// One thread per (row, 32-column group) of a u8 [R][K] pixel matrix: the group becomes 32 bf16
// values (x * scale: the B operand of dW1 = dh^T x) and, for the block-scaled fp8 forward GEMMs,
// 32 e4m3 bytes + one UE8M0 scale byte written into the chunk layout the tensor core consumes
// (epi_common.cuh) and/or their exactly dequantised bf16 values (ddq, the operand the trainer's
// bf16 wgmma reads).  K % 16 == 0, so a group is one or two 16-byte loads.
__device__ __forceinline__ void prep_group(const uint8_t* __restrict__ src, __nv_bfloat16* dbf, uint8_t* dq,
                                           uint8_t* dsf, __nv_bfloat16* ddq, int row, int g, int K, int n_kb,
                                           float scale) {
  const int k0 = g * 32;
  const int n = K - k0 < 32 ? K - k0 : 32;      // 32 or 16
  const long long off = static_cast<long long>(row) * K + k0;
  uint32_t wd[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  {
    const uint4 a = __ldcg(reinterpret_cast<const uint4*>(src + off));   // L2: may have just been DMA'd
    wd[0] = a.x; wd[1] = a.y; wd[2] = a.z; wd[3] = a.w;
    if (n > 16) {
      const uint4 b = __ldcg(reinterpret_cast<const uint4*>(src + off + 16));
      wd[4] = b.x; wd[5] = b.y; wd[6] = b.z; wd[7] = b.w;
    }
  }
  float v[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = static_cast<float>((wd[i >> 2] >> (8 * (i & 3))) & 0xffu) * scale;
  if (dbf != nullptr) {
    uint4* o = reinterpret_cast<uint4*>(dbf + off);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (i * 8 >= n) break;
      o[i] = make_uint4(pack_bf16x2(v[8 * i], v[8 * i + 1]), pack_bf16x2(v[8 * i + 2], v[8 * i + 3]),
                        pack_bf16x2(v[8 * i + 4], v[8 * i + 5]), pack_bf16x2(v[8 * i + 6], v[8 * i + 7]));
    }
  }
  if (dq != nullptr || ddq != nullptr) {
    uint32_t w[8];
    const int e = epi::mx8_quant32(v, w);
    if (dq != nullptr) {
      uint4* o = reinterpret_cast<uint4*>(dq + off);
      o[0] = make_uint4(w[0], w[1], w[2], w[3]);
      if (n > 16) o[1] = make_uint4(w[4], w[5], w[6], w[7]);
      dsf[epi::mx8_sf_index(row, g, n_kb)] = static_cast<uint8_t>(e);
    }
    if (ddq != nullptr) epi::mx8_dq32_store(w, e, ddq + off, n);
  }
}

struct PrepArgs {
  const uint8_t* src; __nv_bfloat16* dbf; uint8_t* dq; uint8_t* dsf; __nv_bfloat16* ddq;
  int R, K; float scale;
  // chunked (input pipeline) variant
  int rows_per_chunk, n_chunks;
  const int* in_flags;       // [n_chunks] written by H2D copies (tag of the data now in src)
  const int* in_seq;         // rounds fed so far; this round's chunks carry tag *in_seq + 1
  unsigned int* cnt;         // [n_chunks] monotonically increasing CTA arrivals
  unsigned int* ready;       // [n_chunks] completed conversions (rounds)
  unsigned int* err;         // set to 1 when a chunk's tag never arrived (host checks it)
};

__global__ void __launch_bounds__(256) k_prep_inputs(PrepArgs a, const int* pred) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  if (pred != nullptr && *pred == 0) return;
  const int G = (a.K + 31) / 32, n_kb = (a.K + 127) / 128;
  const long long total = static_cast<long long>(a.R) * G;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += stride)
    prep_group(a.src, a.dbf, a.dq, a.dsf, a.ddq, static_cast<int>(i / G), static_cast<int>(i % G), a.K, n_kb,
               a.scale);
}

// e4m3 [R][K] + scale chunks -> exact bf16 values, one thread per (row, 32-column group)
__global__ void __launch_bounds__(256) k_mx8_dequant(const uint8_t* __restrict__ q, const uint8_t* __restrict__ sf,
                                                     int R, int K, __nv_bfloat16* __restrict__ dst) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  const int G = (K + 31) / 32, n_kb = (K + 127) / 128;
  const long long total = static_cast<long long>(R) * G;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += stride) {
    const int row = static_cast<int>(i / G), g = static_cast<int>(i % G);
    const int n = K - g * 32 < 32 ? K - g * 32 : 32;
    const long long off = static_cast<long long>(row) * K + g * 32;
    uint32_t w[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const uint4 a = *reinterpret_cast<const uint4*>(q + off);
    w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w;
    if (n > 16) {
      const uint4 b = *reinterpret_cast<const uint4*>(q + off + 16);
      w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
    }
    epi::mx8_dq32_store(w, sf[epi::mx8_sf_index(row, g, n_kb)], dst + off, n);
  }
}

// Input pipeline: the round's uint8 inputs arrive from pinned host memory in `n_chunks` pieces
// (one per local training step), each followed by a 4-byte tag copied on the same copy stream.
// This persistent side-branch kernel converts chunk s as soon as its tag shows up and then
// publishes ready[s] = the tag it converted; the training kernel's TMA producer waits until
// ready[step] reaches the round's tag -- the H2D copy of step s+1..n overlaps the compute
// of step s instead of sitting in front of the whole round.  With no fresh copy (device-only
// rounds) the tags already match and it degenerates to the plain conversion.
// A tag that never arrives (host stalled for seconds between launching the graph and feeding it)
// does not trap -- that would destroy the context and with it the symmetric heap every peer is
// spinning on: the kernel backs off with nanosleep for ~10 s, then sets *err, converts whatever
// is in the buffer and moves on; the host raises after the round.
__global__ void __launch_bounds__(256) k_prep_chunks(PrepArgs a) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  // the round's tag = device round counter + 1: the consensus kernel bumps the counter at the
  // very end of the round (after every reader), the host tags its copies with the same number
  // -- no host -> device copy of a sequence word in front of the graph
  const int want = *reinterpret_cast<const volatile int*>(a.in_seq) + 1;
  const int G = (a.K + 31) / 32, n_kb = (a.K + 127) / 128;
  const long long per = static_cast<long long>(a.rows_per_chunk) * G;
  const long long tid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (int s = 0; s < a.n_chunks; ++s) {
    if (threadIdx.x == 0) {
      unsigned long long spins = 0;
      unsigned int ns = 20;
      while (static_cast<int>(ptx::ld_acquire_sys(reinterpret_cast<const uint32_t*>(a.in_flags + s))) - want < 0) {
        if (++spins > (1ull << 14)) { __nanosleep(ns); if (ns < 2000) ns *= 2; }
        if (spins > (1ull << 14) + 5000000ull) {   // ~10 s of 2 us naps
          if (a.err != nullptr) atomicExch(a.err, 1u);
          break;
        }
      }
    }
    __syncthreads();
    const int row0 = s * a.rows_per_chunk;
    for (long long i = tid; i < per; i += stride)
      prep_group(a.src, a.dbf, a.dq, a.dsf, a.ddq, row0 + static_cast<int>(i / G), static_cast<int>(i % G), a.K,
                 n_kb, a.scale);
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      const unsigned int old = atomicAdd(a.cnt + s, 1u);
      if ((old + 1u) % gridDim.x == 0u)   // last CTA of this pass: chunk s now holds tag `want`
        asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(a.ready + s), "r"(static_cast<unsigned int>(want))
                     : "memory");
    }
  }
}

// fp32 master weights of the 2-layer MLP -> Mx8MlpLayout blob (e4m3 + scale chunks + fp32 biases).
// One thread per (row, K-group) of the PADDED problems; padding rows / groups get scale 1.0
// (0x7F, never NaN) and zero data, so TMA zero-fill and the padded classes contribute nothing.
// dq (optional): the same groups dequantised to bf16, W1 [hidden][in_dim] | W2 [64][hidden].
struct BlobArgs {
  const float* master; long long off_w1, off_b1, off_w2, off_b2;
  int in_dim, hidden, n_classes; uint8_t* blob; Mx8MlpLayout l; __nv_bfloat16* dq;
};
__device__ __forceinline__ void blob_group(const float* w, int ld, int rows, int K, int row, int g, int n_kb,
                                           uint8_t* q, uint8_t* sf, int q_rows, __nv_bfloat16* dq) {
  uint8_t* sfp = sf + epi::mx8_sf_index(row, g, n_kb);
  const int k0 = g * 32;
  if (k0 >= K || row >= q_rows) { *sfp = 127; return; }
  const int n = K - k0 < 32 ? K - k0 : 32;
  float v[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = (row < rows && i < n) ? w[static_cast<long long>(row) * ld + k0 + i] : 0.f;
  uint32_t o[8];
  const int e = epi::mx8_quant32(v, o);
  *sfp = static_cast<uint8_t>(e);
  uint8_t* qp = q + static_cast<long long>(row) * ld + k0;
  for (int i = 0; i < n / 4; ++i) reinterpret_cast<uint32_t*>(qp)[i] = o[i];
  if (dq != nullptr) {
    __nv_bfloat16* d = dq + static_cast<long long>(row) * ld + k0;
    for (int i = 0; i < n / 4; ++i) *reinterpret_cast<uint2*>(d + 4 * i) = epi::mx8_dq4(o[i], e);
  }
}
__global__ void __launch_bounds__(256) k_quantize_mlp_blob(BlobArgs a) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  const int g1 = a.l.kb1 * 4, g2 = a.l.kb2 * 4;
  const int r1 = (a.hidden + 127) / 128 * 128;
  const long long n1 = static_cast<long long>(r1) * g1, n2 = 128LL * g2, n3 = a.hidden + 64;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n1 + n2 + n3; i += stride) {
    if (i < n1) {
      blob_group(a.master + a.off_w1, a.in_dim, a.hidden, a.in_dim, static_cast<int>(i / g1), static_cast<int>(i % g1),
                 a.l.kb1, a.blob + a.l.w1q, a.blob + a.l.w1sf, a.hidden, a.dq);
    } else if (i < n1 + n2) {
      const long long u = i - n1;
      blob_group(a.master + a.off_w2, a.hidden, a.n_classes, a.hidden, static_cast<int>(u / g2), static_cast<int>(u % g2),
                 a.l.kb2, a.blob + a.l.w2q, a.blob + a.l.w2sf, 64,
                 a.dq != nullptr ? a.dq + static_cast<long long>(a.hidden) * a.in_dim : nullptr);
    } else {
      const int u = static_cast<int>(i - n1 - n2);
      float* b = reinterpret_cast<float*>(a.blob + (u < a.hidden ? a.l.b1 + 4 * u : a.l.b2 + 4 * (u - a.hidden)));
      *b = u < a.hidden ? a.master[a.off_b1 + u]
                        : (u - a.hidden < a.n_classes ? a.master[a.off_b2 + u - a.hidden] : 0.f);
    }
  }
}

}  // namespace

#define BFLC_LAUNCH_1D(kernel, nvec, ...)                       \
  do {                                                          \
    (void)cudaGetLastError(); /* drop a stale error of this thread */ \
    kernel<<<grid_for(nvec), kBlock, 0, s>>>(__VA_ARGS__);      \
    note_launch();                                              \
    return cudaGetLastError();                                  \
  } while (0)

#define BFLC_LAUNCH_1D_PDL(kernel, nvec, ...)                                          \
  do {                                                                                \
    note_launch();                                                                    \
    return launch_pdl(kernel, dim3(grid_for(nvec)), dim3(kBlock), 0, s, __VA_ARGS__); \
  } while (0)

cudaError_t cast_f32_to_bf16(const float* src, void* dst, int64_t n, cudaStream_t s) {
  BFLC_LAUNCH_1D(k_cast_f32_bf16, n / 8 + 1, src, reinterpret_cast<__nv_bfloat16*>(dst), n);
}
cudaError_t cast_bf16_to_f32(const void* src, float* dst, int64_t n, cudaStream_t s) {
  BFLC_LAUNCH_1D(k_cast_bf16_f32, n, reinterpret_cast<const __nv_bfloat16*>(src), dst, n);
}
cudaError_t prep_inputs_u8(const uint8_t* src, void* dst_bf16, void* dst_q, uint8_t* dst_sf, int R,
                           int K, float scale, cudaStream_t s, void* dst_dq) {
  if (K % 16 != 0 || R <= 0 || (dst_q != nullptr && dst_sf == nullptr)) return cudaErrorInvalidValue;
  PrepArgs a{};
  a.src = src; a.dbf = reinterpret_cast<__nv_bfloat16*>(dst_bf16); a.dq = static_cast<uint8_t*>(dst_q);
  a.dsf = dst_sf; a.ddq = static_cast<__nv_bfloat16*>(dst_dq); a.R = R; a.K = K; a.scale = scale;
  const long long total = static_cast<long long>(R) * ((K + 31) / 32);
  note_launch();
  return launch_pdl(k_prep_inputs, dim3(grid_for(total)), dim3(kBlock), 0, s, a, current_predicate());
}
cudaError_t prep_inputs_u8_chunks(const uint8_t* src, void* dst_bf16, void* dst_q, uint8_t* dst_sf,
                                  int rows_per_chunk, int K, int n_chunks, float scale,
                                  const int* in_flags, const int* in_seq, unsigned int* cnt,
                                  unsigned int* ready, unsigned int* err, cudaStream_t s, void* dst_dq) {
  if (K % 16 != 0 || n_chunks <= 0 || rows_per_chunk <= 0 || (dst_q != nullptr && dst_sf == nullptr))
    return cudaErrorInvalidValue;
  PrepArgs a{};
  a.src = src; a.dbf = reinterpret_cast<__nv_bfloat16*>(dst_bf16); a.dq = static_cast<uint8_t*>(dst_q);
  a.dsf = dst_sf; a.ddq = static_cast<__nv_bfloat16*>(dst_dq); a.R = rows_per_chunk * n_chunks; a.K = K; a.scale = scale;
  a.rows_per_chunk = rows_per_chunk; a.n_chunks = n_chunks;
  a.in_flags = in_flags; a.in_seq = in_seq; a.cnt = cnt; a.ready = ready; a.err = err;
  note_launch();
  return launch_pdl(k_prep_chunks, dim3(16), dim3(256), 0, s, a);
}
cudaError_t quantize_mlp_blob(const float* master, long long off_w1, long long off_b1,
                              long long off_w2, long long off_b2, int in_dim, int hidden,
                              int n_classes, uint8_t* blob, cudaStream_t s, void* dq) {
  if (in_dim % 4 != 0 || hidden % 4 != 0 || n_classes > 64) return cudaErrorInvalidValue;
  BlobArgs a{master, off_w1, off_b1, off_w2, off_b2, in_dim, hidden, n_classes, blob,
             mx8_mlp_layout(in_dim, hidden), static_cast<__nv_bfloat16*>(dq)};
  const long long total = static_cast<long long>((hidden + 127) / 128 * 128) * a.l.kb1 * 4 + 128LL * a.l.kb2 * 4 +
                          hidden + 64;
  note_launch();
  return launch_pdl(k_quantize_mlp_blob, dim3(grid_for(total)), dim3(kBlock), 0, s, a);
}
cudaError_t mx8_dequant_bf16(const void* q, const uint8_t* sf, int R, int K, void* dst, cudaStream_t s) {
  if (K % 16 != 0 || R <= 0) return cudaErrorInvalidValue;
  note_launch();
  return launch_pdl(k_mx8_dequant, dim3(grid_for(static_cast<long long>(R) * ((K + 31) / 32))), dim3(kBlock), 0, s,
                    static_cast<const uint8_t*>(q), sf, R, K, static_cast<__nv_bfloat16*>(dst));
}
cudaError_t cast_u8_to_bf16(const uint8_t* src, void* dst, int64_t n, float scale,
                            cudaStream_t s) {
  BFLC_LAUNCH_1D_PDL(k_cast_u8_bf16, n / 16 + 1, src, reinterpret_cast<__nv_bfloat16*>(dst), n,
                     scale, current_predicate());
}
cudaError_t quantize_fp8(const void* src_bf16, uint8_t* dst, int64_t n, float inv_scale,
                         cudaStream_t s) {
  BFLC_LAUNCH_1D(k_quant_fp8, n / 8 + 1, reinterpret_cast<const __nv_bfloat16*>(src_bf16), dst, n,
                 inv_scale);
}
cudaError_t amax_bf16(const void* src, int64_t n, float* amax_out, cudaStream_t s) {
  BFLC_LAUNCH_1D(k_amax_bf16, n, reinterpret_cast<const __nv_bfloat16*>(src), n, amax_out);
}
cudaError_t fill_f32(float* dst, int64_t n, float v, cudaStream_t s) {
  BFLC_LAUNCH_1D(k_fill, n, dst, n, v);
}
cudaError_t add_bf16(const void* a, const void* b, void* out, int64_t n, cudaStream_t s) {
  BFLC_LAUNCH_1D(k_add_bf16, n / 8 + 1, reinterpret_cast<const __nv_bfloat16*>(a),
                 reinterpret_cast<const __nv_bfloat16*>(b), reinterpret_cast<__nv_bfloat16*>(out),
                 n);
}
cudaError_t sgd_step(const OptimArgs& a, cudaStream_t s) {
  BFLC_LAUNCH_1D_PDL(k_optim<false>, a.n / 4 + 1, a);
}
cudaError_t adam_step(const OptimArgs& a, cudaStream_t s) {
  if (!a.m || !a.v) return cudaErrorInvalidValue;
  BFLC_LAUNCH_1D_PDL(k_optim<true>, a.n / 4 + 1, a);
}

static bool recipe_ok(const RecipeArgs& a) {
  if (a.schedule < kLrConstant || a.schedule > kLrCosine || a.warmup < 0 || a.total < 0 || !(a.decay >= 0.f))
    return false;
  if (a.schedule != kLrConstant && a.total <= a.warmup) return false;
  return a.decay == 0.f || a.no_decay != nullptr;
}
cudaError_t sgd_recipe_step(const RecipeArgs& a, cudaStream_t s) {
  if (!recipe_ok(a)) return cudaErrorInvalidValue;
  BFLC_LAUNCH_1D_PDL((k_optim<false, true>), a.n / 4 + 1, a);
}
cudaError_t adam_recipe_step(const RecipeArgs& a, cudaStream_t s) {
  if (!a.m || !a.v || !recipe_ok(a)) return cudaErrorInvalidValue;
  BFLC_LAUNCH_1D_PDL((k_optim<true, true>), a.n / 4 + 1, a);
}
cudaError_t grad_norm_f32(const float* grad, int64_t n, void* workspace, float* norm_out, float max_norm,
                          int* skipped, const int* active, cudaStream_t s) {
  if (workspace == nullptr || norm_out == nullptr || n <= 0) return cudaErrorInvalidValue;
  NormArgs a{grad, n, static_cast<GradNormState*>(workspace),
             reinterpret_cast<double*>(static_cast<char*>(workspace) + sizeof(GradNormState)), norm_out,
             max_norm, skipped, active};
  static_assert(sizeof(GradNormState) % 8 == 0, "partials must be 8-byte aligned");
  BFLC_LAUNCH_1D_PDL(k_grad_norm, n / 4 + 1, a);
}

}  // namespace bflc
