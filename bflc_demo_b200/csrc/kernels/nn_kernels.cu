// Non-GEMM layers for the CNN / transformer model families (LeNet-5, ResNet-18, BERT-base):
// im2col / col2im (convolutions run as wgmma GEMMs over the column matrix), pooling,
// batch-norm, layer-norm, row softmax, embeddings, head transposes.  All tensors are bf16,
// channels-last (NHWC) for images so a convolution's GEMM output IS the next layer's input;
// statistics and parameter gradients are fp32.
//
// The reference has none of these (its only model is x@W+b, python-sdk/main.py:113-120);
// they exist because BASELINE.json names LeNet-5 / ResNet-18 / BERT-base configs.
#include <cuda_bf16.h>

#include "bflc_kernels.h"
#include "philox.hpp"

namespace bflc {

namespace {

constexpr int kT = 256;
typedef __nv_bfloat16 bf16;

inline int blocks_for(int64_t n, int per = kT, int cap = 132 * 16) {
  int64_t g = (n + per - 1) / per;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<int>(g);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// block-wide sum broadcast to all threads (blockDim.x == kT)
__device__ __forceinline__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float t = (threadIdx.x < kT / 32) ? sh[threadIdx.x] : 0.f;
  if (w == 0) {
    t = warp_sum(t);
    if (l == 0) sh[0] = t;
  }
  __syncthreads();
  return sh[0];
}

// ------------------------------------------------------------------ im2col / col2im
// x: [N, H, W, C] -> col: [N*OH*OW, ld_col], column index = (kh*KW + kw)*C + c
__global__ void k_im2col(const bf16* __restrict__ x, bf16* __restrict__ col, int N, int C, int H,
                         int W, int KH, int KW, int stride, int pad, int OH, int OW,
                         long long ld_col) {
  const long long kcols = static_cast<long long>(KH) * KW * C;
  const long long total = static_cast<long long>(N) * OH * OW * kcols;
  const long long step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += step) {
    const long long row = i / kcols;
    const int kc = static_cast<int>(i - row * kcols);
    const int c = kc % C;
    const int kw = (kc / C) % KW;
    const int kh = kc / (C * KW);
    const int ow = static_cast<int>(row % OW);
    const int oh = static_cast<int>((row / OW) % OH);
    const int n = static_cast<int>(row / (static_cast<long long>(OW) * OH));
    const int ih = oh * stride - pad + kh, iw = ow * stride - pad + kw;
    bf16 v = __float2bfloat16(0.f);
    if (ih >= 0 && ih < H && iw >= 0 && iw < W)
      v = x[((static_cast<long long>(n) * H + ih) * W + iw) * C + c];
    col[row * ld_col + kc] = v;
  }
}

// Zero-stuffed upsampling of a strided convolution's output gradient: up[n, s*oh, s*ow, :] =
// dy[n, oh, ow, :], zero elsewhere.  The input gradient of a stride-s convolution is then the
// stride-1 implicit-GEMM convolution of `up` (ConvView flip mode).  8 channels (16 B) per thread.
__global__ void k_upsample_zero(const uint4* __restrict__ dy, uint4* __restrict__ up, int N, int H,
                                int W, int OH, int OW, int C8, int stride) {
  const long long total = static_cast<long long>(N) * H * W * C8;
  const long long step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += step) {
    const int c = static_cast<int>(i % C8);
    const long long pix = i / C8;
    const int iw = static_cast<int>(pix % W);
    const int ih = static_cast<int>((pix / W) % H);
    const int n = static_cast<int>(pix / (static_cast<long long>(W) * H));
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    const int oh = ih / stride, ow = iw / stride;
    if (oh * stride == ih && ow * stride == iw && oh < OH && ow < OW)
      v = dy[((static_cast<long long>(n) * OH + oh) * OW + ow) * C8 + c];
    up[i] = v;
  }
}

// gather form of the transpose: each dx element sums the col entries it was copied to
__global__ void k_col2im(const bf16* __restrict__ col, bf16* __restrict__ dx, int N, int C, int H,
                         int W, int KH, int KW, int stride, int pad, int OH, int OW,
                         long long ld_col) {
  const long long total = static_cast<long long>(N) * H * W * C;
  const long long step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += step) {
    const int c = static_cast<int>(i % C);
    const int w = static_cast<int>((i / C) % W);
    const int h = static_cast<int>((i / (static_cast<long long>(C) * W)) % H);
    const int n = static_cast<int>(i / (static_cast<long long>(C) * W * H));
    float acc = 0.f;
    for (int kh = 0; kh < KH; ++kh) {
      const int t = h + pad - kh;
      if (t < 0 || t % stride) continue;
      const int oh = t / stride;
      if (oh >= OH) continue;
      for (int kw = 0; kw < KW; ++kw) {
        const int u = w + pad - kw;
        if (u < 0 || u % stride) continue;
        const int ow = u / stride;
        if (ow >= OW) continue;
        const long long row = (static_cast<long long>(n) * OH + oh) * OW + ow;
        acc += __bfloat162float(col[row * ld_col + (kh * KW + kw) * C + c]);
      }
    }
    dx[i] = __float2bfloat16(acc);
  }
}

// ------------------------------------------------------------------ pooling (NHWC)
__global__ void k_maxpool_fwd(const bf16* __restrict__ x, bf16* __restrict__ y,
                              int32_t* __restrict__ idx, int N, int C, int H, int W, int k,
                              int stride, int pad, int OH, int OW) {
  const long long total = static_cast<long long>(N) * OH * OW * C;
  const long long step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += step) {
    const int c = static_cast<int>(i % C);
    const int ow = static_cast<int>((i / C) % OW);
    const int oh = static_cast<int>((i / (static_cast<long long>(C) * OW)) % OH);
    const int n = static_cast<int>(i / (static_cast<long long>(C) * OW * OH));
    float best = -INFINITY;
    int bi = -1;
    for (int a = 0; a < k; ++a)
      for (int b = 0; b < k; ++b) {
        const int ih = oh * stride - pad + a, iw = ow * stride - pad + b;
        if (ih < 0 || ih >= H || iw < 0 || iw >= W) continue;
        const long long src = ((static_cast<long long>(n) * H + ih) * W + iw) * C + c;
        const float v = __bfloat162float(x[src]);
        if (v > best) { best = v; bi = static_cast<int>(src % (static_cast<long long>(H) * W * C)); }
      }
    y[i] = __float2bfloat16(best);
    idx[i] = bi;  // offset inside sample n
  }
}
// dx must be zeroed by the caller; windows may overlap (ResNet stem: k=3, stride=2)
__global__ void k_maxpool_bwd(const bf16* __restrict__ dy, const int32_t* __restrict__ idx,
                              float* __restrict__ dx_f32, long long n_out, long long per_out,
                              long long per_in) {
  const long long step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n_out;
       i += step) {
    const long long n = i / per_out;
    const int j = idx[i];
    if (j >= 0) atomicAdd(dx_f32 + n * per_in + j, __bfloat162float(dy[i]));
  }
}

__global__ void k_avgpool_fwd(const bf16* __restrict__ x, bf16* __restrict__ y, int N, int HW,
                              int C) {
  const long long total = static_cast<long long>(N) * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    const long long n = i / C;
    float s = 0.f;
    for (int p = 0; p < HW; ++p) s += __bfloat162float(x[(n * HW + p) * C + c]);
    y[i] = __float2bfloat16(s / HW);
  }
}
__global__ void k_avgpool_bwd(const bf16* __restrict__ dy, bf16* __restrict__ dx, int N, int HW,
                              int C) {
  const long long total = static_cast<long long>(N) * HW * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    const long long n = i / (static_cast<long long>(HW) * C);
    dx[i] = __float2bfloat16(__bfloat162float(dy[n * C + c]) / HW);
  }
}

// ------------------------------------------------------------------ batch norm [rows][C]
// stats: each block owns a slab of rows and a tile of 32 channels x 8 row-lanes.  The sums are
// of x - x[0, c] (shifted by the channel's first row): sum(x^2)/rows - mean^2 in fp32 loses the
// variance of channels whose |mean| is large against their std (on an H100, a channel of mean 100
// and std 0.5 over 16384 rows got rstd 3.4e-3 off); around a sample of the channel the two terms
// stay comparable.
__global__ void k_bn_stats(const bf16* __restrict__ x, float* __restrict__ sum,
                           float* __restrict__ sumsq, long long rows, int C) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int lane_r = threadIdx.x >> 5;  // 0..7
  float s = 0.f, q = 0.f;
  if (c < C) {
    const float pivot = __bfloat162float(x[c]);
    for (long long r = blockIdx.y * 8 + lane_r; r < rows; r += static_cast<long long>(gridDim.y) * 8) {
      const float v = __bfloat162float(x[r * C + c]) - pivot;
      s += v; q += v * v;
    }
  }
  __shared__ float shs[8][33], shq[8][33];
  shs[lane_r][threadIdx.x & 31] = s;
  shq[lane_r][threadIdx.x & 31] = q;
  __syncthreads();
  if (lane_r == 0 && c < C) {
#pragma unroll
    for (int k = 1; k < 8; ++k) { s += shs[k][threadIdx.x & 31]; q += shq[k][threadIdx.x & 31]; }
    atomicAdd(sum + c, s);
    atomicAdd(sumsq + c, q);
  }
}
// mean / rstd hold the shifted sums of k_bn_stats on entry
__global__ void k_bn_finalize(const bf16* __restrict__ x, float* mean, float* rstd, float* run_mean,
                              float* run_var, long long rows, int C, float eps, float momentum) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float d = mean[c] / rows;
  const float m = __bfloat162float(x[c]) + d;
  float var = rstd[c] / rows - d * d;
  var = fmaxf(var, 0.f);
  mean[c] = m;
  rstd[c] = rsqrtf(var + eps);
  if (run_mean) {
    run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * m;
    const float unb = rows > 1 ? var * rows / (rows - 1) : var;
    run_var[c] = (1.f - momentum) * run_var[c] + momentum * unb;
  }
}
__global__ void k_bn_apply(const bf16* __restrict__ x, bf16* __restrict__ y,
                           const float* __restrict__ gamma, const float* __restrict__ beta,
                           const float* __restrict__ mean, const float* __restrict__ rstd,
                           const bf16* __restrict__ residual, long long total, int C, int relu) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    float v = (__bfloat162float(x[i]) - mean[c]) * rstd[c] * gamma[c] + beta[c];
    if (residual) v += __bfloat162float(residual[i]);
    if (relu) v = fmaxf(v, 0.f);
    y[i] = __float2bfloat16(v);
  }
}
// backward pass 1: dgamma = sum g*xhat, dbeta = sum g   (g = dy masked by relu)
__global__ void k_bn_bwd_reduce(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                const bf16* __restrict__ y, const float* __restrict__ mean,
                                const float* __restrict__ rstd, float* __restrict__ dgamma,
                                float* __restrict__ dbeta, long long rows, int C, int relu) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int lane_r = threadIdx.x >> 5;
  float sg = 0.f, sb = 0.f;
  if (c < C) {
    const float m = mean[c], rs = rstd[c];
    for (long long r = blockIdx.y * 8 + lane_r; r < rows; r += static_cast<long long>(gridDim.y) * 8) {
      float g = __bfloat162float(dy[r * C + c]);
      if (relu && !(__bfloat162float(y[r * C + c]) > 0.f)) g = 0.f;
      sg += g * (__bfloat162float(x[r * C + c]) - m) * rs;
      sb += g;
    }
  }
  __shared__ float s1[8][33], s2[8][33];
  s1[lane_r][threadIdx.x & 31] = sg;
  s2[lane_r][threadIdx.x & 31] = sb;
  __syncthreads();
  if (lane_r == 0 && c < C) {
#pragma unroll
    for (int k = 1; k < 8; ++k) { sg += s1[k][threadIdx.x & 31]; sb += s2[k][threadIdx.x & 31]; }
    atomicAdd(dgamma + c, sg);
    atomicAdd(dbeta + c, sb);
  }
}
__global__ void k_bn_bwd_apply(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                               const bf16* __restrict__ y, const float* __restrict__ gamma,
                               const float* __restrict__ mean, const float* __restrict__ rstd,
                               const float* __restrict__ dgamma, const float* __restrict__ dbeta,
                               bf16* __restrict__ dx, bf16* __restrict__ dres, long long rows,
                               int C, int relu) {
  const long long total = rows * C;
  const float inv = 1.f / rows;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    float g = __bfloat162float(dy[i]);
    if (relu && !(__bfloat162float(y[i]) > 0.f)) g = 0.f;
    if (dres) dres[i] = __float2bfloat16(g);
    const float xhat = (__bfloat162float(x[i]) - mean[c]) * rstd[c];
    dx[i] = __float2bfloat16(gamma[c] * rstd[c] * (g - inv * (dbeta[c] + xhat * dgamma[c])));
  }
}

// ------------------------------------------------------------------ group norm [N * HW][C]
// One block per (example n, group g): the group is the HW rows of example n times its cg = C / G
// channels [g * cg, (g + 1) * cg).  Its statistics never mix examples, so an example's output and
// gradients depend on that example alone (DP-SGD needs this; batch norm cannot give it).  Element e of
// the group is row e / cg, channel e % cg.  Every sum runs in a fixed order: the layer is
// bit-reproducible, its parameter gradients included.
__device__ __forceinline__ long long gn_at(long long base, int e, int cg, int C) {
  const int r = e / cg;
  return base + static_cast<long long>(r) * C + (e - r * cg);
}

// mean and variance in two passes (the variance of x - mean, not E[x^2] - mean^2)
__global__ void __launch_bounds__(kT) k_gn_fwd(const bf16* __restrict__ x, bf16* __restrict__ y,
                                               const float* __restrict__ gamma, const float* __restrict__ beta,
                                               float* __restrict__ mean, float* __restrict__ rstd,
                                               const bf16* __restrict__ residual, int HW, int C, int cg,
                                               float eps, int relu) {
  __shared__ float sh[kT / 32];
  const int G = C / cg, n = blockIdx.x / G, g = blockIdx.x - n * G, M = HW * cg;
  const long long base = static_cast<long long>(n) * HW * C + static_cast<long long>(g) * cg;
  float s = 0.f;
  for (int e = threadIdx.x; e < M; e += kT) s += __bfloat162float(x[gn_at(base, e, cg, C)]);
  // correctly rounded even under --use_fast_math, as in k_ln_fwd: a constant group sees x - m == 0
  const float m = __fdiv_rn(block_sum(s, sh), static_cast<float>(M));
  float q = 0.f;
  for (int e = threadIdx.x; e < M; e += kT) {
    const float d = __bfloat162float(x[gn_at(base, e, cg, C)]) - m;
    q = fmaf(d, d, q);
  }
  const float rs = rsqrtf(__fdiv_rn(block_sum(q, sh), static_cast<float>(M)) + eps);
  if (threadIdx.x == 0) {
    mean[blockIdx.x] = m;
    rstd[blockIdx.x] = rs;
  }
  for (int e = threadIdx.x; e < M; e += kT) {
    const long long i = gn_at(base, e, cg, C);
    const int c = g * cg + e % cg;
    float v = (__bfloat162float(x[i]) - m) * rs * gamma[c] + beta[c];
    if (residual) v += __bfloat162float(residual[i]);
    if (relu) v = fmaxf(v, 0.f);
    y[i] = __float2bfloat16(v);
  }
}

// g = dy masked by the ReLU; per channel c of the group: pg[n, c] = sum_t g xhat, pb[n, c] = sum_t g
// (this example's own dgamma / dbeta), then dx = rstd (gamma_c g - mean(gamma g) - xhat mean(gamma g xhat))
// over the group, and dres = g.  Channel partials: thread t takes channel t % cw of a chunk of cw =
// min(cg, kT) channels and rows t / cw, t / cw + nl, ... (nl = kT / cw lanes); the lanes are summed in order.
__global__ void __launch_bounds__(kT) k_gn_bwd(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                               const bf16* __restrict__ y, const float* __restrict__ gamma,
                                               const float* __restrict__ mean, const float* __restrict__ rstd,
                                               bf16* __restrict__ dx, bf16* __restrict__ dres,
                                               float* __restrict__ pg, float* __restrict__ pb, int HW, int C,
                                               int cg, int relu) {
  __shared__ float sh[kT / 32];
  __shared__ float sa[kT], sb[kT];
  const int G = C / cg, n = blockIdx.x / G, g = blockIdx.x - n * G, M = HW * cg;
  const long long base = static_cast<long long>(n) * HW * C + static_cast<long long>(g) * cg;
  const float m = mean[blockIdx.x], rs = rstd[blockIdx.x];
  const int cw = cg < kT ? cg : kT, nl = kT / cw, ct = threadIdx.x % cw, lane = threadIdx.x / cw;
  float s1 = 0.f, s2 = 0.f;
  for (int c0 = 0; c0 < cg; c0 += cw) {
    const int c = c0 + ct;
    float a = 0.f, b = 0.f;
    if (lane < nl && c < cg) {
      for (int r = lane; r < HW; r += nl) {
        const long long i = base + static_cast<long long>(r) * C + c;
        float gv = __bfloat162float(dy[i]);
        if (relu && !(__bfloat162float(y[i]) > 0.f)) gv = 0.f;
        a = fmaf(gv, (__bfloat162float(x[i]) - m) * rs, a);
        b += gv;
      }
      const float gm = gamma[g * cg + c];
      s1 = fmaf(gm, b, s1);
      s2 = fmaf(gm, a, s2);
    }
    sa[threadIdx.x] = a;
    sb[threadIdx.x] = b;
    __syncthreads();
    if (threadIdx.x < cw && c < cg) {
      float ta = 0.f, tb = 0.f;
      for (int l = 0; l < nl; ++l) {
        ta += sa[l * cw + threadIdx.x];
        tb += sb[l * cw + threadIdx.x];
      }
      pg[static_cast<long long>(n) * C + g * cg + c] = ta;
      pb[static_cast<long long>(n) * C + g * cg + c] = tb;
    }
    __syncthreads();
  }
  const float inv = __fdiv_rn(1.f, static_cast<float>(M));
  s1 = block_sum(s1, sh) * inv;
  s2 = block_sum(s2, sh) * inv;
  for (int e = threadIdx.x; e < M; e += kT) {
    const long long i = gn_at(base, e, cg, C);
    float gv = __bfloat162float(dy[i]);
    if (relu && !(__bfloat162float(y[i]) > 0.f)) gv = 0.f;
    if (dres) dres[i] = __float2bfloat16(gv);
    const float xh = (__bfloat162float(x[i]) - m) * rs;
    dx[i] = __float2bfloat16(rs * (gamma[g * cg + e % cg] * gv - s1 - xh * s2));
  }
}

// dgamma[c] += sum_n pg[n, c], dbeta[c] += sum_n pb[n, c], examples in order.  With a per-example factor
// cf (DP-SGD's clip factors): the terms are cf[n] pg[n, c] (one rounding each, no contraction), and an
// example whose factor is 0 is skipped -- a dropped example's partials may not be finite
__global__ void k_gn_param(const float* __restrict__ pg, const float* __restrict__ pb, float* __restrict__ dgamma,
                           float* __restrict__ dbeta, int N, int C, const float* __restrict__ cf) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float a = 0.f, b = 0.f;
  if (cf == nullptr) {
    for (int n = 0; n < N; ++n) {
      a += pg[static_cast<long long>(n) * C + c];
      b += pb[static_cast<long long>(n) * C + c];
    }
  } else {
    for (int n = 0; n < N; ++n) {
      const float f = cf[n];
      if (f == 0.f) continue;
      a = __fadd_rn(a, __fmul_rn(f, pg[static_cast<long long>(n) * C + c]));
      b = __fadd_rn(b, __fmul_rn(f, pb[static_cast<long long>(n) * C + c]));
    }
  }
  dgamma[c] += a;
  dbeta[c] += b;
}

// ------------------------------------------------------------------ layer norm [rows][C]
__global__ void __launch_bounds__(kT) k_ln_fwd(const bf16* __restrict__ x, bf16* __restrict__ y,
                                               const float* __restrict__ gamma,
                                               const float* __restrict__ beta,
                                               float* __restrict__ mean, float* __restrict__ rstd,
                                               long long rows, int C, float eps) {
  __shared__ float sh[kT / 32];
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    const bf16* xr = x + r * C;
    float s = 0.f;
    for (int c = threadIdx.x; c < C; c += kT) s += __bfloat162float(xr[c]);
    // correctly rounded even under --use_fast_math: a constant row must see x - m == 0 exactly, or
    // eps = 1e-12 turns a one-ulp error of m into xhat of order 0.1
    const float m = __fdiv_rn(block_sum(s, sh), static_cast<float>(C));
    float q = 0.f;
    for (int c = threadIdx.x; c < C; c += kT) {
      const float d = __bfloat162float(xr[c]) - m;
      q += d * d;
    }
    const float rs = rsqrtf(block_sum(q, sh) / C + eps);
    if (threadIdx.x == 0) { mean[r] = m; rstd[r] = rs; }
    for (int c = threadIdx.x; c < C; c += kT)
      y[r * C + c] = __float2bfloat16((__bfloat162float(xr[c]) - m) * rs * gamma[c] + beta[c]);
  }
}
// C <= 4 * kT.  Each block walks a strided set of rows and keeps per-column partial
// dgamma/dbeta in registers -> one atomic per column per block.
__global__ void __launch_bounds__(kT) k_ln_bwd(const bf16* __restrict__ dy,
                                               const bf16* __restrict__ x,
                                               const float* __restrict__ gamma,
                                               const float* __restrict__ mean,
                                               const float* __restrict__ rstd,
                                               bf16* __restrict__ dx, float* __restrict__ dgamma,
                                               float* __restrict__ dbeta, long long rows, int C) {
  __shared__ float sh[kT / 32];
  float pg[4] = {0.f, 0.f, 0.f, 0.f}, pb[4] = {0.f, 0.f, 0.f, 0.f};
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    const float m = mean[r], rs = rstd[r];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = threadIdx.x + k * kT;
      if (c < C) {
        const float g = __bfloat162float(dy[r * C + c]);
        const float xh = (__bfloat162float(x[r * C + c]) - m) * rs;
        pg[k] += g * xh;
        pb[k] += g;
        const float gg = g * gamma[c];
        s1 += gg;
        s2 += gg * xh;
      }
    }
    s1 = block_sum(s1, sh) / C;
    s2 = block_sum(s2, sh) / C;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = threadIdx.x + k * kT;
      if (c < C) {
        const float g = __bfloat162float(dy[r * C + c]) * gamma[c];
        const float xh = (__bfloat162float(x[r * C + c]) - m) * rs;
        dx[r * C + c] = __float2bfloat16(rs * (g - s1 - xh * s2));
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = threadIdx.x + k * kT;
    if (c < C) { atomicAdd(dgamma + c, pg[k]); atomicAdd(dbeta + c, pb[k]); }
  }
}

// ------------------------------------------------------------------ row softmax (one warp/row)
__global__ void k_softmax_fwd(const bf16* __restrict__ x, bf16* __restrict__ y, long long rows,
                              int cols, float scale) {
  const long long r = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int l = threadIdx.x & 31;
  if (r >= rows) return;
  float mx = -INFINITY;
  for (int c = l; c < cols; c += 32) mx = fmaxf(mx, __bfloat162float(x[r * cols + c]) * scale);
  mx = warp_max(mx);
  float s = 0.f;
  for (int c = l; c < cols; c += 32) s += __expf(__bfloat162float(x[r * cols + c]) * scale - mx);
  s = 1.f / warp_sum(s);
  for (int c = l; c < cols; c += 32)
    y[r * cols + c] = __float2bfloat16(__expf(__bfloat162float(x[r * cols + c]) * scale - mx) * s);
}
__global__ void k_softmax_bwd(const bf16* __restrict__ dy, const bf16* __restrict__ y,
                              bf16* __restrict__ dx, long long rows, int cols, float scale) {
  const long long r = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int l = threadIdx.x & 31;
  if (r >= rows) return;
  float dot = 0.f;
  for (int c = l; c < cols; c += 32)
    dot += __bfloat162float(dy[r * cols + c]) * __bfloat162float(y[r * cols + c]);
  dot = warp_sum(dot);
  for (int c = l; c < cols; c += 32) {
    const float p = __bfloat162float(y[r * cols + c]);
    dx[r * cols + c] = __float2bfloat16(scale * p * (__bfloat162float(dy[r * cols + c]) - dot));
  }
}

// ------------------------------------------------------------------ embeddings
__global__ void k_embed_fwd(const int32_t* __restrict__ ids, const bf16* __restrict__ table,
                            const bf16* __restrict__ pos, bf16* __restrict__ out, long long rows,
                            int seq, int C, const int32_t* __restrict__ pos_ids) {
  const long long total = rows * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / C;
    const int c = static_cast<int>(i - r * C);
    float v = __bfloat162float(table[static_cast<long long>(ids[r]) * C + c]);
    if (pos) v += __bfloat162float(pos[static_cast<long long>(pos_ids ? pos_ids[r] : r % seq) * C + c]);
    out[i] = __float2bfloat16(v);
  }
}
__global__ void k_embed_bwd(const int32_t* __restrict__ ids, const bf16* __restrict__ dy,
                            float* __restrict__ dtable, float* __restrict__ dpos, long long rows,
                            int seq, int C, const int32_t* __restrict__ pos_ids) {
  const long long total = rows * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / C;
    const int c = static_cast<int>(i - r * C);
    const float g = __bfloat162float(dy[i]);
    atomicAdd(dtable + static_cast<long long>(ids[r]) * C + c, g);
    if (dpos) atomicAdd(dpos + static_cast<long long>(pos_ids ? pos_ids[r] : r % seq) * C + c, g);
  }
}

// [d0][d1][d2][d3] -> [d0][d2][d1][d3]
__global__ void k_transpose_0213(const bf16* __restrict__ x, bf16* __restrict__ y, int d0, int d1,
                                 int d2, int d3) {
  const long long total = static_cast<long long>(d0) * d1 * d2 * d3;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int e = static_cast<int>(i % d3);
    const int b = static_cast<int>((i / d3) % d1);
    const int c = static_cast<int>((i / (static_cast<long long>(d3) * d1)) % d2);
    const long long a = i / (static_cast<long long>(d3) * d1 * d2);
    // i indexes the OUTPUT [a][c][b][e]
    y[i] = x[((a * d1 + b) * d2 + c) * d3 + e];
  }
}

// dz = dy * act'(aux) and colsum[c] += sum_rows dz   (mode 0: identity, 1: ReLU with aux = y,
// 2: GELU with aux = pre-activation).  Tile: 32 channels x 8 row-lanes per block.
__global__ void k_act_bwd_colsum(const bf16* __restrict__ dy, const bf16* __restrict__ aux,
                                 bf16* __restrict__ dz, float* __restrict__ colsum, long long rows,
                                 int C, int mode) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int lane_r = threadIdx.x >> 5;
  float s = 0.f;
  if (c < C) {
    for (long long r = blockIdx.y * 8 + lane_r; r < rows; r += static_cast<long long>(gridDim.y) * 8) {
      float g = __bfloat162float(dy[r * C + c]);
      if (mode == 1) {
        if (!(__bfloat162float(aux[r * C + c]) > 0.f)) g = 0.f;
      } else if (mode == 2) {
        const float x = __bfloat162float(aux[r * C + c]);
        const float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752f));
        g *= cdf + x * 0.3989422804014327f * __expf(-0.5f * x * x);
      }
      if (dz) dz[r * C + c] = __float2bfloat16(g);
      s += g;
    }
  }
  __shared__ float sh[8][33];
  sh[lane_r][threadIdx.x & 31] = s;
  __syncthreads();
  if (lane_r == 0 && c < C && colsum) {
#pragma unroll
    for (int k = 1; k < 8; ++k) s += sh[k][threadIdx.x & 31];
    atomicAdd(colsum + c, s);
  }
}

// ------------------------------------------------------------------ dropout (philox.hpp)
__device__ __forceinline__ philox::Drop drop_at(philox::Drop d, const int32_t* step) {
  d.step += static_cast<uint32_t>(*step);   // d.step holds the host step add
  return d;
}

// y = (x +) z * keep / (1 - p), 8 columns (one Philox call, 16 B) per thread
__global__ void k_dropout_add(const bf16* __restrict__ x, const bf16* __restrict__ z, bf16* __restrict__ y,
                              long long rows, int C8, int S, const int32_t* __restrict__ seq_ids,
                              const int32_t* __restrict__ pos_ids, philox::Drop d, const int32_t* step) {
  d = drop_at(d, step);
  const long long total = rows * C8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / C8;
    const int g = static_cast<int>(i - r * C8);
    const uint32_t seq = seq_ids ? static_cast<uint32_t>(seq_ids[r]) : static_cast<uint32_t>(r / S);
    const uint32_t pos = seq_ids ? static_cast<uint32_t>(pos_ids[r]) : static_cast<uint32_t>(r % S);
    const uint32_t bits = philox::keep8(d, seq, 0, pos, g);
    const uint4 zv = reinterpret_cast<const uint4*>(z)[i];
    const uint4 xv = x ? reinterpret_cast<const uint4*>(x)[i] : make_uint4(0u, 0u, 0u, 0u);
    const uint32_t zw[4] = {zv.x, zv.y, zv.z, zv.w}, xw[4] = {xv.x, xv.y, xv.z, xv.w};
    uint32_t out[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 zf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&zw[t]));
      const float2 xf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&xw[t]));
      const float a = xf.x + ((bits >> (2 * t)) & 1u ? zf.x * d.scale : 0.f);
      const float b = xf.y + ((bits >> (2 * t + 1)) & 1u ? zf.y * d.scale : 0.f);
      const __nv_bfloat162 o = __floats2bfloat162_rn(a, b);
      out[t] = *reinterpret_cast<const uint32_t*>(&o);
    }
    reinterpret_cast<uint4*>(y)[i] = make_uint4(out[0], out[1], out[2], out[3]);
  }
}

// keep mask of attention dropout, uint8 [B*H, S, S]: one thread per (b, h, row, 8 columns)
__global__ void k_dropout_keep_mask(uint8_t* __restrict__ mask, int H, int S, long long total,
                                    philox::Drop d, const int32_t* step) {
  d = drop_at(d, step);
  const int S8 = S / 8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % S8);
    const int row = static_cast<int>((i / S8) % S);
    const long long bh = i / (static_cast<long long>(S8) * S);
    const uint32_t bits = philox::keep8(d, static_cast<uint32_t>(bh / H), static_cast<uint32_t>(bh % H), row, g);
    uint2 v;
    v.x = (bits & 1u) | ((bits >> 1) & 1u) << 8 | ((bits >> 2) & 1u) << 16 | ((bits >> 3) & 1u) << 24;
    v.y = ((bits >> 4) & 1u) | ((bits >> 5) & 1u) << 8 | ((bits >> 6) & 1u) << 16 | ((bits >> 7) & 1u) << 24;
    reinterpret_cast<uint2*>(mask)[i] = v;
  }
}

// -> false for arguments the dropout kernels cannot take
bool drop_params(const DropoutArgs& a, philox::Drop& d) {
  if (!(a.p > 0.f && a.p < 1.f) || a.step == nullptr || a.site >= (1u << 24)) return false;
  d.seed_lo = static_cast<uint32_t>(a.seed);
  d.seed_hi = static_cast<uint32_t>(a.seed >> 32);
  d.step = static_cast<uint32_t>(a.step_add);
  d.site = a.site;
  d.thr = philox::threshold(a.p);
  d.scale = 1.f / (1.f - a.p);
  return true;
}


// ------------------------------------------------------------------ vocabulary-wide cross-entropy
// One CTA per row of fp32 logits [M, ld] with V valid columns.  Each thread scans columns
// tid, tid + kT, ... (float4 groups, then the V % 4 tail) keeping an online (max, sum exp) and the
// first index of its maximum; the CTA combines them in a fixed shuffle / smem tree, so loss and
// dlogits are bit-reproducible.  Argmax ties go to the lowest column, as in the GEMM ARGMAX_ACC
// epilogue (a strict > scan in column order).
struct XentPart {
  float m, s;
  int idx;
};
__device__ __forceinline__ void xent_take(XentPart& a, float x, int c) {
  if (x > a.m) {
    a.s = a.s * __expf(a.m - x) + 1.f;   // a.m = -inf: 0 * ... + 1
    a.m = x;
    a.idx = c;
  } else {
    a.s += __expf(x - a.m);
  }
}
__device__ __forceinline__ XentPart xent_merge(XentPart a, XentPart b) {
  const float m = fmaxf(a.m, b.m);
  XentPart r;
  r.m = m;
  r.s = (a.m == -INFINITY ? 0.f : a.s * __expf(a.m - m)) + (b.m == -INFINITY ? 0.f : b.s * __expf(b.m - m));
  r.idx = a.m > b.m ? a.idx : b.m > a.m ? b.idx : min(a.idx, b.idx);
  return r;
}
__device__ __forceinline__ XentPart xent_shfl(XentPart a, int o) {
  XentPart b;
  b.m = __shfl_xor_sync(0xffffffffu, a.m, o);
  b.s = __shfl_xor_sync(0xffffffffu, a.s, o);
  b.idx = __shfl_xor_sync(0xffffffffu, a.idx, o);
  return xent_merge(a, b);
}

__global__ void __launch_bounds__(kT) k_xent_rows(const float* __restrict__ logits, int V, long long ld,
                                                  const int32_t* __restrict__ targets, float* __restrict__ loss,
                                                  int32_t* __restrict__ hits, bf16* __restrict__ dl, long long ldd,
                                                  float grad_scale) {
  __shared__ XentPart sh[kT / 32];
  const long long row = blockIdx.x;
  const float* z = logits + row * ld;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  XentPart a{-INFINITY, 0.f, -1};
  const int n4 = V >> 2;
  for (int c4 = tid; c4 < n4; c4 += kT) {
    const float4 v = reinterpret_cast<const float4*>(z)[c4];
    xent_take(a, v.x, 4 * c4);
    xent_take(a, v.y, 4 * c4 + 1);
    xent_take(a, v.z, 4 * c4 + 2);
    xent_take(a, v.w, 4 * c4 + 3);
  }
  if (tid < V - 4 * n4) xent_take(a, z[4 * n4 + tid], 4 * n4 + tid);
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) a = xent_shfl(a, o);
  if (lane == 0) sh[w] = a;
  __syncthreads();
  XentPart t = sh[0];
#pragma unroll
  for (int i = 1; i < kT / 32; ++i) t = xent_merge(t, sh[i]);
  const int32_t tgt = targets[row];
  const bool tgt_ok = tgt >= 0 && tgt < V;
  if (tid == 0) {
    if (loss != nullptr) loss[row] = tgt_ok ? t.m + __logf(t.s) - z[tgt] : __int_as_float(0x7fc00000);
    if (hits != nullptr && tgt_ok && t.idx == tgt) atomicAdd(hits, 1);
  }
  if (dl == nullptr) return;
  // dlogits = (softmax - onehot) * grad_scale, pad columns [V, ldd) = 0
  const float inv = 1.f / t.s;
  bf16* d = dl + row * ldd;
  for (long long c = tid; c < ldd; c += kT) {
    float g = 0.f;
    if (c < V) g = (__expf(z[c] - t.m) * inv - (c == tgt ? 1.f : 0.f)) * grad_scale;
    d[c] = __float2bfloat16(g);
  }
}

}  // namespace

cudaError_t act_bwd_colsum(const void* dy, const void* aux, void* dz, float* colsum, int64_t rows,
                           int C, int mode, cudaStream_t s) {
  dim3 g((C + 31) / 32, static_cast<unsigned>(rows / 64 > 128 ? 128 : (rows / 64 > 0 ? rows / 64 : 1)));
  (void)cudaGetLastError();
  k_act_bwd_colsum<<<g, kT, 0, s>>>(reinterpret_cast<const bf16*>(dy),
                                    reinterpret_cast<const bf16*>(aux), reinterpret_cast<bf16*>(dz),
                                    colsum, rows, C, mode);
  note_launch();
  return cudaGetLastError();
}

#define NN_LAUNCH(kernel, grid, ...)            \
  do {                                          \
    (void)cudaGetLastError(); /* drop a stale error of this thread */ \
    kernel<<<grid, kT, 0, s>>>(__VA_ARGS__);    \
    note_launch();                              \
    return cudaGetLastError();                  \
  } while (0)

cudaError_t im2col_bf16(const void* x, void* col, int N, int C, int H, int W, int KH, int KW,
                        int stride, int pad, int OH, int OW, int64_t ld_col, cudaStream_t s) {
  const int64_t total = static_cast<int64_t>(N) * OH * OW * KH * KW * C;
  NN_LAUNCH(k_im2col, blocks_for(total), reinterpret_cast<const bf16*>(x),
            reinterpret_cast<bf16*>(col), N, C, H, W, KH, KW, stride, pad, OH, OW, ld_col);
}
cudaError_t col2im_bf16(const void* col, void* dx, int N, int C, int H, int W, int KH, int KW,
                        int stride, int pad, int OH, int OW, int64_t ld_col, cudaStream_t s) {
  NN_LAUNCH(k_col2im, blocks_for(static_cast<int64_t>(N) * H * W * C),
            reinterpret_cast<const bf16*>(col), reinterpret_cast<bf16*>(dx), N, C, H, W, KH, KW,
            stride, pad, OH, OW, ld_col);
}
cudaError_t upsample_zero_bf16(const void* dy, void* up, int N, int H, int W, int OH, int OW, int C,
                               int stride, cudaStream_t s) {
  if (C % 8 != 0) return cudaErrorInvalidValue;
  NN_LAUNCH(k_upsample_zero, blocks_for(static_cast<int64_t>(N) * H * W * (C / 8)),
            reinterpret_cast<const uint4*>(dy), reinterpret_cast<uint4*>(up), N, H, W, OH, OW, C / 8,
            stride);
}
cudaError_t maxpool2d_fwd(const void* x, void* y, int32_t* idx, int N, int C, int H, int W, int k,
                          int stride, int pad, int OH, int OW, cudaStream_t s) {
  NN_LAUNCH(k_maxpool_fwd, blocks_for(static_cast<int64_t>(N) * OH * OW * C),
            reinterpret_cast<const bf16*>(x), reinterpret_cast<bf16*>(y), idx, N, C, H, W, k, stride,
            pad, OH, OW);
}
// dx_f32: fp32 scratch [N * per_in] zeroed by the caller (overlapping windows accumulate);
// n_out = N * per_out
cudaError_t maxpool2d_bwd(const void* dy, const int32_t* idx, float* dx_f32, int64_t n_out,
                          int64_t per_out, int64_t per_in, cudaStream_t s) {
  NN_LAUNCH(k_maxpool_bwd, blocks_for(n_out), reinterpret_cast<const bf16*>(dy), idx, dx_f32, n_out,
            per_out, per_in);
}
cudaError_t avgpool_global_fwd(const void* x, void* y, int N, int HW, int C, cudaStream_t s) {
  NN_LAUNCH(k_avgpool_fwd, blocks_for(static_cast<int64_t>(N) * C), reinterpret_cast<const bf16*>(x),
            reinterpret_cast<bf16*>(y), N, HW, C);
}
cudaError_t avgpool_global_bwd(const void* dy, void* dx, int N, int HW, int C, cudaStream_t s) {
  NN_LAUNCH(k_avgpool_bwd, blocks_for(static_cast<int64_t>(N) * HW * C),
            reinterpret_cast<const bf16*>(dy), reinterpret_cast<bf16*>(dx), N, HW, C);
}

cudaError_t batchnorm_fwd(const void* x, void* y, const float* gamma, const float* beta,
                          float* mean, float* rstd, float* run_mean, float* run_var,
                          int64_t rows, int C, float eps, float momentum, int training, int relu,
                          const void* residual, cudaStream_t s) {
  if (training) {
    cudaError_t e = cudaMemsetAsync(mean, 0, sizeof(float) * C, s);
    if (e != cudaSuccess) return e;
    e = cudaMemsetAsync(rstd, 0, sizeof(float) * C, s);
    if (e != cudaSuccess) return e;
    dim3 g((C + 31) / 32, static_cast<unsigned>(rows / 64 > 64 ? 64 : (rows / 64 > 0 ? rows / 64 : 1)));
    (void)cudaGetLastError();
    k_bn_stats<<<g, kT, 0, s>>>(reinterpret_cast<const bf16*>(x), mean, rstd, rows, C);
    note_launch();
    k_bn_finalize<<<(C + 127) / 128, 128, 0, s>>>(reinterpret_cast<const bf16*>(x), mean, rstd,
                                                   run_mean, run_var, rows, C, eps, momentum);
    note_launch();
  }
  NN_LAUNCH(k_bn_apply, blocks_for(rows * C), reinterpret_cast<const bf16*>(x),
            reinterpret_cast<bf16*>(y), gamma, beta, mean, rstd,
            reinterpret_cast<const bf16*>(residual), rows * C, C, relu);
}
cudaError_t batchnorm_bwd(const void* dy, const void* x, const void* y, const float* gamma,
                          const float* mean, const float* rstd, void* dx, float* dgamma,
                          float* dbeta, void* dresidual, int64_t rows, int C, int relu,
                          cudaStream_t s) {
  // dgamma / dbeta are accumulation targets (flat gradient buffer): the statistics of THIS call
  // must be isolated, so reduce into them only when they are zero on entry (the optimizer zeroes
  // the gradient buffer every step) -- documented contract.
  dim3 g((C + 31) / 32, static_cast<unsigned>(rows / 64 > 64 ? 64 : (rows / 64 > 0 ? rows / 64 : 1)));
  (void)cudaGetLastError();
  k_bn_bwd_reduce<<<g, kT, 0, s>>>(reinterpret_cast<const bf16*>(dy), reinterpret_cast<const bf16*>(x),
                                   reinterpret_cast<const bf16*>(y), mean, rstd, dgamma, dbeta, rows,
                                   C, relu);
  note_launch();
  NN_LAUNCH(k_bn_bwd_apply, blocks_for(rows * C), reinterpret_cast<const bf16*>(dy),
            reinterpret_cast<const bf16*>(x), reinterpret_cast<const bf16*>(y), gamma, mean, rstd,
            dgamma, dbeta, reinterpret_cast<bf16*>(dx), reinterpret_cast<bf16*>(dresidual), rows, C,
            relu);
}

namespace {
bool gn_shape_ok(int N, int HW, int C, int G) {
  return N >= 1 && HW >= 1 && G >= 1 && C >= G && C % G == 0 &&
         static_cast<int64_t>(HW) * (C / G) <= INT32_MAX && static_cast<int64_t>(N) * G <= INT32_MAX;
}
}  // namespace

cudaError_t groupnorm_fwd(const void* x, void* y, const float* gamma, const float* beta, float* mean,
                          float* rstd, int N, int HW, int C, int G, float eps, int relu,
                          const void* residual, cudaStream_t s) {
  if (!gn_shape_ok(N, HW, C, G)) return cudaErrorInvalidValue;
  NN_LAUNCH(k_gn_fwd, N * G, reinterpret_cast<const bf16*>(x), reinterpret_cast<bf16*>(y), gamma, beta,
            mean, rstd, reinterpret_cast<const bf16*>(residual), HW, C, C / G, eps, relu);
}
cudaError_t groupnorm_bwd(const void* dy, const void* x, const void* y, const float* gamma,
                          const float* mean, const float* rstd, void* dx, float* dgamma, float* dbeta,
                          void* dresidual, float* pg, float* pb, int N, int HW, int C, int G, int relu,
                          cudaStream_t s) {
  if (!gn_shape_ok(N, HW, C, G)) return cudaErrorInvalidValue;
  (void)cudaGetLastError();
  k_gn_bwd<<<N * G, kT, 0, s>>>(reinterpret_cast<const bf16*>(dy), reinterpret_cast<const bf16*>(x),
                                reinterpret_cast<const bf16*>(y), gamma, mean, rstd, reinterpret_cast<bf16*>(dx),
                                reinterpret_cast<bf16*>(dresidual), pg, pb, HW, C, C / G, relu);
  note_launch();
  k_gn_param<<<(C + 127) / 128, 128, 0, s>>>(pg, pb, dgamma, dbeta, N, C, nullptr);
  note_launch();
  return cudaGetLastError();
}
cudaError_t groupnorm_param(const float* pg, const float* pb, float* dgamma, float* dbeta, int N, int C,
                            const float* cf, cudaStream_t s) {
  if (N < 1 || C < 1) return cudaErrorInvalidValue;
  (void)cudaGetLastError();
  k_gn_param<<<(C + 127) / 128, 128, 0, s>>>(pg, pb, dgamma, dbeta, N, C, cf);
  note_launch();
  return cudaGetLastError();
}

cudaError_t layernorm_fwd(const void* x, const void* residual, void* y, const float* gamma,
                          const float* beta, float* mean, float* rstd, int64_t rows, int C,
                          float eps, cudaStream_t s) {
  if (residual != nullptr) return cudaErrorNotSupported;  // add with add_bf16 first
  const int grid = static_cast<int>(rows < 132 * 8 ? rows : 132 * 8);
  NN_LAUNCH(k_ln_fwd, grid, reinterpret_cast<const bf16*>(x), reinterpret_cast<bf16*>(y), gamma, beta,
            mean, rstd, rows, C, eps);
}
cudaError_t layernorm_bwd(const void* dy, const void* xin, const float* gamma, const float* mean,
                          const float* rstd, void* dx, float* dgamma, float* dbeta, int64_t rows,
                          int C, cudaStream_t s) {
  if (C > 4 * kT) return cudaErrorInvalidValue;
  const int grid = static_cast<int>(rows < 132 * 2 ? rows : 132 * 2);
  NN_LAUNCH(k_ln_bwd, grid, reinterpret_cast<const bf16*>(dy), reinterpret_cast<const bf16*>(xin),
            gamma, mean, rstd, reinterpret_cast<bf16*>(dx), dgamma, dbeta, rows, C);
}
cudaError_t softmax_rows_fwd(const void* x, void* y, int64_t rows, int cols, float scale,
                             cudaStream_t s) {
  NN_LAUNCH(k_softmax_fwd, static_cast<int>((rows * 32 + kT - 1) / kT),
            reinterpret_cast<const bf16*>(x), reinterpret_cast<bf16*>(y), rows, cols, scale);
}
cudaError_t softmax_rows_bwd(const void* dy, const void* y, void* dx, int64_t rows, int cols,
                             float scale, cudaStream_t s) {
  NN_LAUNCH(k_softmax_bwd, static_cast<int>((rows * 32 + kT - 1) / kT),
            reinterpret_cast<const bf16*>(dy), reinterpret_cast<const bf16*>(y),
            reinterpret_cast<bf16*>(dx), rows, cols, scale);
}
cudaError_t embedding_fwd(const int32_t* ids, const void* table_bf16, const void* pos_bf16,
                          void* out, int64_t rows, int seq, int C, cudaStream_t s, const int32_t* pos_ids) {
  NN_LAUNCH(k_embed_fwd, blocks_for(rows * C), ids, reinterpret_cast<const bf16*>(table_bf16),
            reinterpret_cast<const bf16*>(pos_bf16), reinterpret_cast<bf16*>(out), rows, seq, C, pos_ids);
}
cudaError_t embedding_bwd(const int32_t* ids, const void* dy, float* dtable, float* dpos,
                          int64_t rows, int seq, int C, cudaStream_t s, const int32_t* pos_ids) {
  NN_LAUNCH(k_embed_bwd, blocks_for(rows * C), ids, reinterpret_cast<const bf16*>(dy), dtable, dpos,
            rows, seq, C, pos_ids);
}
cudaError_t transpose_0213_bf16(const void* x, void* y, int d0, int d1, int d2, int d3,
                                cudaStream_t s) {
  NN_LAUNCH(k_transpose_0213, blocks_for(static_cast<int64_t>(d0) * d1 * d2 * d3),
            reinterpret_cast<const bf16*>(x), reinterpret_cast<bf16*>(y), d0, d1, d2, d3);
}

cudaError_t dropout_add_bf16(const void* x, const void* z, void* y, int64_t rows, int C, int S,
                             const int32_t* seq_ids, const int32_t* pos_ids, const DropoutArgs& drop,
                             cudaStream_t s) {
  philox::Drop d{};
  if (!drop_params(drop, d) || C % 8 != 0 || rows < 0 || (seq_ids == nullptr && S <= 0) ||
      (seq_ids != nullptr && pos_ids == nullptr))
    return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  NN_LAUNCH(k_dropout_add, blocks_for(rows * (C / 8)), reinterpret_cast<const bf16*>(x),
            reinterpret_cast<const bf16*>(z), reinterpret_cast<bf16*>(y), rows, C / 8, S, seq_ids, pos_ids, d,
            drop.step);
}

cudaError_t dropout_keep_mask(uint8_t* mask, int B, int H, int S, const DropoutArgs& drop, cudaStream_t s) {
  philox::Drop d{};
  if (!drop_params(drop, d) || B <= 0 || H <= 0 || S <= 0 || S % 8 != 0) return cudaErrorInvalidValue;
  const long long total = static_cast<long long>(B) * H * S * (S / 8);
  NN_LAUNCH(k_dropout_keep_mask, blocks_for(total), mask, H, S, total, d, drop.step);
}

cudaError_t xent_rows(const float* logits, int64_t M, int V, int64_t ld, const int32_t* targets, float* loss,
                      int32_t* hits, void* dlogits, int64_t ldd, float grad_scale, cudaStream_t s) {
  if (logits == nullptr || targets == nullptr || M < 0 || M > INT32_MAX || V < 1 || ld < V || ld % 4 != 0 ||
      reinterpret_cast<uintptr_t>(logits) % 16 != 0 || (dlogits != nullptr && ldd < V))
    return cudaErrorInvalidValue;
  if (M == 0) return cudaSuccess;
  NN_LAUNCH(k_xent_rows, static_cast<int>(M), logits, V, static_cast<long long>(ld), targets, loss, hits,
            reinterpret_cast<bf16*>(dlogits), static_cast<long long>(ldd), grad_scale);
}

}  // namespace bflc
