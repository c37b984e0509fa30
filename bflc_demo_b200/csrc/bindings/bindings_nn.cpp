// Bindings for the non-GEMM NN kernels (csrc/kernels/nn_kernels.cu).
#include <ATen/cuda/CUDAContext.h>
#include <torch/extension.h>

#include <optional>

#include "bflc_kernels.h"

namespace py = pybind11;
using OptT = std::optional<at::Tensor>;

namespace {
void check(cudaError_t e, const char* what) {
  TORCH_CHECK(e == cudaSuccess, "bflc::", what, " failed: ", cudaGetErrorString(e));
}
cudaStream_t st() { return at::cuda::getCurrentCUDAStream().stream(); }
template <typename T>
T* optp(const OptT& t) { return t.has_value() ? reinterpret_cast<T*>(t->data_ptr()) : nullptr; }
void check_lengths(const OptT& lengths, const at::Tensor& q, int B) {
  if (!lengths.has_value()) return;
  TORCH_CHECK(lengths->scalar_type() == at::kInt && lengths->is_contiguous() && lengths->numel() == B &&
                  lengths->device() == q.device(),
              "attention: lengths must be a contiguous int32 tensor of B elements on q's device");
}
void check_pos_ids(const OptT& pos_ids, const at::Tensor& ids, int64_t rows) {
  if (!pos_ids.has_value()) return;
  TORCH_CHECK(pos_ids->scalar_type() == at::kInt && pos_ids->is_contiguous() && pos_ids->numel() == rows &&
                  pos_ids->device() == ids.device(),
              "embedding: pos_ids must be a contiguous int32 tensor of one position per row on ids' device");
}
// packed attention: cu_seqlens int32 [B+1] on q's device, max_seqlen in [1, 512]; -> S_pad
int64_t check_packed(const at::Tensor& cu, const at::Tensor& q, int64_t max_seqlen) {
  TORCH_CHECK(cu.scalar_type() == at::kInt && cu.is_contiguous() && cu.dim() == 1 && cu.numel() >= 2 &&
                  cu.device() == q.device(),
              "attention_packed: cu_seqlens must be a contiguous int32 tensor of B+1 elements on q's device");
  TORCH_CHECK(max_seqlen >= 1 && max_seqlen <= 512, "attention_packed: max_seqlen must lie in [1, 512], got ",
              max_seqlen);
  return (max_seqlen + 63) / 64 * 64;
}
void check_workspace(const at::Tensor& t, const at::Tensor& q, int64_t n, const char* what) {
  TORCH_CHECK(t.scalar_type() == at::kFloat && t.is_contiguous() && t.numel() >= n && t.device() == q.device(),
              "attention_packed: ", what, " must be a contiguous fp32 tensor of at least B*H*S_pad = ", n,
              " elements on q's device");
}
// dropout arguments (philox.hpp): p in [0, 1), 0 = off; p > 0 needs the step word, an int32 tensor of
// one element on `like`'s device; site in [0, 2^24)
bflc::DropoutArgs dropout_args(double p, uint64_t seed, const OptT& step, int64_t step_add, int64_t site,
                               const at::Tensor& like, const char* who) {
  TORCH_CHECK(p >= 0.0 && p < 1.0 && static_cast<float>(p) < 1.f, who, ": dropout_p must lie in [0, 1), got ", p);
  bflc::DropoutArgs d;
  if (p == 0.0) return d;
  TORCH_CHECK(step.has_value() && step->scalar_type() == at::kInt && step->is_contiguous() && step->numel() == 1 &&
                  step->device() == like.device(),
              who, ": dropout needs a step word: a contiguous int32 tensor of one element on the operands' device");
  TORCH_CHECK(site >= 0 && site < (1 << 24), who, ": dropout site must lie in [0, 2^24), got ", site);
  TORCH_CHECK(step_add >= INT32_MIN && step_add <= INT32_MAX, who, ": step_add must fit in int32");
  d.p = static_cast<float>(p);
  d.seed = seed;
  d.step = step->data_ptr<int32_t>();
  d.step_add = static_cast<int>(step_add);
  d.site = static_cast<uint32_t>(site);
  return d;
}
}  // namespace

void bind_nn(py::module_& m) {
  m.def("im2col", [](at::Tensor x, at::Tensor col, int N, int C, int H, int W, int KH, int KW,
                     int stride, int pad, int OH, int OW) {
    check(bflc::im2col_bf16(x.data_ptr(), col.data_ptr(), N, C, H, W, KH, KW, stride, pad, OH, OW,
                            col.stride(0), st()), "im2col");
  });
  m.def("col2im", [](at::Tensor col, at::Tensor dx, int N, int C, int H, int W, int KH, int KW,
                     int stride, int pad, int OH, int OW) {
    check(bflc::col2im_bf16(col.data_ptr(), dx.data_ptr(), N, C, H, W, KH, KW, stride, pad, OH, OW,
                            col.stride(0), st()), "col2im");
  });
  m.def("upsample_zero", [](at::Tensor dy, at::Tensor up, int N, int H, int W, int OH, int OW, int Cc,
                            int stride) {
    check(bflc::upsample_zero_bf16(dy.data_ptr(), up.data_ptr(), N, H, W, OH, OW, Cc, stride, st()),
          "upsample_zero");
  });
  m.def("maxpool_fwd", [](at::Tensor x, at::Tensor y, at::Tensor idx, int N, int C, int H, int W,
                          int k, int stride, int pad, int OH, int OW) {
    check(bflc::maxpool2d_fwd(x.data_ptr(), y.data_ptr(), idx.data_ptr<int32_t>(), N, C, H, W, k,
                              stride, pad, OH, OW, st()), "maxpool_fwd");
  });
  m.def("maxpool_bwd", [](at::Tensor dy, at::Tensor idx, at::Tensor dx_f32, int64_t per_out,
                          int64_t per_in) {
    check(bflc::maxpool2d_bwd(dy.data_ptr(), idx.data_ptr<int32_t>(), dx_f32.data_ptr<float>(),
                              dy.numel(), per_out, per_in, st()), "maxpool_bwd");
  });
  m.def("avgpool_fwd", [](at::Tensor x, at::Tensor y, int N, int HW, int C) {
    check(bflc::avgpool_global_fwd(x.data_ptr(), y.data_ptr(), N, HW, C, st()), "avgpool_fwd");
  });
  m.def("avgpool_bwd", [](at::Tensor dy, at::Tensor dx, int N, int HW, int C) {
    check(bflc::avgpool_global_bwd(dy.data_ptr(), dx.data_ptr(), N, HW, C, st()), "avgpool_bwd");
  });
  m.def("batchnorm_fwd", [](at::Tensor x, at::Tensor y, at::Tensor gamma, at::Tensor beta,
                            at::Tensor mean, at::Tensor rstd, const OptT& run_mean,
                            const OptT& run_var, int64_t rows, int C, double eps, double momentum,
                            bool training, bool relu, const OptT& residual) {
    check(bflc::batchnorm_fwd(x.data_ptr(), y.data_ptr(), gamma.data_ptr<float>(),
                              beta.data_ptr<float>(), mean.data_ptr<float>(), rstd.data_ptr<float>(),
                              optp<float>(run_mean), optp<float>(run_var), rows, C, (float)eps,
                              (float)momentum, training, relu,
                              residual.has_value() ? residual->data_ptr() : nullptr, st()),
          "batchnorm_fwd");
  });
  m.def("batchnorm_bwd", [](at::Tensor dy, at::Tensor x, at::Tensor y, at::Tensor gamma,
                            at::Tensor mean, at::Tensor rstd, at::Tensor dx, at::Tensor dgamma,
                            at::Tensor dbeta, const OptT& dres, int64_t rows, int C, bool relu) {
    check(bflc::batchnorm_bwd(dy.data_ptr(), x.data_ptr(), y.data_ptr(), gamma.data_ptr<float>(),
                              mean.data_ptr<float>(), rstd.data_ptr<float>(), dx.data_ptr(),
                              dgamma.data_ptr<float>(), dbeta.data_ptr<float>(),
                              dres.has_value() ? dres->data_ptr() : nullptr, rows, C, relu, st()),
          "batchnorm_bwd");
  });
  m.def("layernorm_fwd", [](at::Tensor x, at::Tensor y, at::Tensor gamma, at::Tensor beta,
                            at::Tensor mean, at::Tensor rstd, int64_t rows, int C, double eps) {
    check(bflc::layernorm_fwd(x.data_ptr(), nullptr, y.data_ptr(), gamma.data_ptr<float>(),
                              beta.data_ptr<float>(), mean.data_ptr<float>(), rstd.data_ptr<float>(),
                              rows, C, (float)eps, st()), "layernorm_fwd");
  });
  m.def("layernorm_bwd", [](at::Tensor dy, at::Tensor x, at::Tensor gamma, at::Tensor mean,
                            at::Tensor rstd, at::Tensor dx, at::Tensor dgamma, at::Tensor dbeta,
                            int64_t rows, int C) {
    check(bflc::layernorm_bwd(dy.data_ptr(), x.data_ptr(), gamma.data_ptr<float>(),
                              mean.data_ptr<float>(), rstd.data_ptr<float>(), dx.data_ptr(),
                              dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), rows, C, st()),
          "layernorm_bwd");
  });
  m.def("softmax_fwd", [](at::Tensor x, at::Tensor y, int64_t rows, int cols, double scale) {
    check(bflc::softmax_rows_fwd(x.data_ptr(), y.data_ptr(), rows, cols, (float)scale, st()),
          "softmax_fwd");
  });
  m.def("softmax_bwd", [](at::Tensor dy, at::Tensor y, at::Tensor dx, int64_t rows, int cols,
                          double scale) {
    check(bflc::softmax_rows_bwd(dy.data_ptr(), y.data_ptr(), dx.data_ptr(), rows, cols,
                                 (float)scale, st()), "softmax_bwd");
  });
  // pos_ids (optional): int32 [rows] position of each row (packed sequences); None: row % seq
  m.def("embedding_fwd", [](at::Tensor ids, at::Tensor table, const OptT& pos, at::Tensor out,
                            int64_t rows, int seq, int C, const OptT& pos_ids) {
    check_pos_ids(pos_ids, ids, rows);
    check(bflc::embedding_fwd(ids.data_ptr<int32_t>(), table.data_ptr(),
                              pos.has_value() ? pos->data_ptr() : nullptr, out.data_ptr(), rows, seq,
                              C, st(), optp<const int32_t>(pos_ids)), "embedding_fwd");
  }, py::arg("ids"), py::arg("table"), py::arg("pos"), py::arg("out"), py::arg("rows"), py::arg("seq"),
     py::arg("C"), py::arg("pos_ids") = py::none());
  m.def("embedding_bwd", [](at::Tensor ids, at::Tensor dy, at::Tensor dtable, const OptT& dpos,
                            int64_t rows, int seq, int C, const OptT& pos_ids) {
    check_pos_ids(pos_ids, ids, rows);
    check(bflc::embedding_bwd(ids.data_ptr<int32_t>(), dy.data_ptr(), dtable.data_ptr<float>(),
                              optp<float>(dpos), rows, seq, C, st(), optp<const int32_t>(pos_ids)),
          "embedding_bwd");
  }, py::arg("ids"), py::arg("dy"), py::arg("dtable"), py::arg("dpos"), py::arg("rows"), py::arg("seq"),
     py::arg("C"), py::arg("pos_ids") = py::none());
  m.def("act_bwd_colsum", [](at::Tensor dy, const OptT& aux, const OptT& dz, const OptT& colsum,
                             int64_t rows, int C, int mode) {
    check(bflc::act_bwd_colsum(dy.data_ptr(), aux.has_value() ? aux->data_ptr() : nullptr,
                               dz.has_value() ? dz->data_ptr() : nullptr, optp<float>(colsum), rows,
                               C, mode, st()), "act_bwd_colsum");
  });
  // ---- block-scaled fp8 (MXFP8) ----
  m.def("mx8_sf_bytes", [](int64_t rows, int64_t K) { return bflc::mx8_sf_bytes((int)rows, (int)K); });
  m.def("quantize_mx8", [](at::Tensor x, at::Tensor q, at::Tensor sf, int64_t R, int64_t K,
                           double in_scale) {
    bflc::DType dt = x.scalar_type() == at::kFloat      ? bflc::DType::F32
                     : x.scalar_type() == at::kBFloat16 ? bflc::DType::BF16
                                                        : bflc::DType::U8;
    TORCH_CHECK(x.scalar_type() == at::kFloat || x.scalar_type() == at::kBFloat16 ||
                    x.scalar_type() == at::kByte, "quantize_mx8: f32 / bf16 / u8 input");
    TORCH_CHECK(x.stride(-1) == 1 && q.stride(-1) == 1, "quantize_mx8: contiguous rows");
    TORCH_CHECK(sf.numel() >= bflc::mx8_sf_bytes((int)R, (int)K), "quantize_mx8: sf buffer too small");
    check(bflc::quantize_mx8(x.data_ptr(), dt, x.stride(0), (int)R, (int)K, (float)in_scale,
                             q.data_ptr(), q.stride(0), sf.data_ptr(), st()), "quantize_mx8");
  });
  m.def("gemm_mx8", [](at::Tensor a, at::Tensor sfa, at::Tensor b, at::Tensor sfb, at::Tensor d,
                       int64_t M, int64_t N, int64_t K, double alpha, const OptT& bias, int64_t act) {
    bflc::Mx8Problem p;
    p.M = (int)M; p.N = (int)N; p.K = (int)K;
    p.a = a.data_ptr(); p.lda = a.stride(0); p.sfa = static_cast<const uint8_t*>(sfa.data_ptr());
    p.b = b.data_ptr(); p.ldb = b.stride(0); p.sfb = static_cast<const uint8_t*>(sfb.data_ptr());
    TORCH_CHECK(sfa.numel() >= bflc::mx8_sf_bytes(p.M, p.K) && sfb.numel() >= bflc::mx8_sf_bytes(p.N, p.K),
                "gemm_mx8: scale-factor buffers too small");
    p.d = d.data_ptr();
    p.d_dtype = d.scalar_type() == at::kFloat ? bflc::DType::F32 : bflc::DType::BF16;
    p.ldd = d.stride(0);
    p.alpha = (float)alpha;
    p.bias = optp<const float>(bias);
    p.act = static_cast<bflc::Act>(act);
    check(bflc::gemm_mx8_sm100(p, st()), "gemm_mx8_sm100");
  });
  // fused attention (seq 128, head dim 64): q, k, v, o, gradients are [B*S, H*64] bf16
  // Implicit-GEMM convolution (ConvView in bflc_kernels.h).  `x` is the NHWC activation the
  // shifted boxes are read from, `other` the dense operand (weights, or dy for mode 2).
  m.def("conv_gemm", [](int mode, int flip, at::Tensor x, at::Tensor other, at::Tensor d, int N, int H,
                        int W, int Cc, int OH, int OW, int KH, int KW, int stride, int pad, int n_out,
                        const OptT& bias, int act, const OptT& aux_out, const OptT& aux_in, int act_bwd,
                        const OptT& colsum, int split_k, bool accumulate) {
    bflc::GemmProblem p;
    auto& cv = p.conv;
    cv.mode = mode; cv.flip = flip; cv.x = x.data_ptr();
    cv.N = N; cv.H = H; cv.W = W; cv.C = Cc; cv.OH = OH; cv.OW = OW;
    cv.KH = KH; cv.KW = KW; cv.stride = stride; cv.pad = pad;
    const int taps = KH * KW;
    const int64_t pixels = (int64_t)N * OH * OW;
    if (mode == 1) {
      p.M = (int)pixels; p.N = n_out; p.K = taps * Cc;
      p.a = {x.data_ptr(), Cc, 0, false};
      p.b = {other.data_ptr(), other.stride(0), 0, flip != 0};
    } else {
      p.M = n_out; p.N = taps * Cc; p.K = (int)pixels;
      p.a = {other.data_ptr(), other.stride(0), 0, true};   // dy [pixels][Cout]
      p.b = {x.data_ptr(), Cc, 0, true};
    }
    auto& e = p.epi;
    e.d = d.data_ptr();
    e.d_dtype = d.scalar_type() == at::kFloat ? bflc::DType::F32 : bflc::DType::BF16;
    e.ldd = d.stride(0);
    e.bias = optp<const float>(bias);
    e.act = static_cast<bflc::Act>(act);
    e.aux_out = aux_out.has_value() ? aux_out->data_ptr() : nullptr;
    e.aux_in = aux_in.has_value() ? aux_in->data_ptr() : nullptr;
    e.act_bwd = act_bwd;
    e.colsum = optp<float>(colsum);
    e.split_k = split_k;
    e.accumulate = accumulate ? 1 : 0;
    check(bflc::gemm_sm100(p, st()), "conv_gemm (implicit-GEMM convolution)");
  });
  // lengths (optional): int32 [B] valid key count per sequence (right-padding mask)
  // dropout_p, seed, step, step_add, site (optional): attention-probability dropout (tiled kernels)
  m.def("attention_fwd", [](at::Tensor q, at::Tensor k, at::Tensor v, at::Tensor o, at::Tensor lse, int B,
                            int S, int H, double scale, const OptT& lengths, double dropout_p, uint64_t seed,
                            const OptT& step, int64_t step_add, int64_t site, bool causal) {
    const int D = (int)q.size(1) / H;
    TORCH_CHECK(q.stride(1) == 1 && k.stride(1) == 1 && v.stride(1) == 1 && o.stride(1) == 1 &&
                q.stride(0) == k.stride(0) && q.stride(0) == v.stride(0) && q.stride(0) == o.stride(0),
                "attention: q, k, v, o must share one row pitch");
    check_lengths(lengths, q, B);
    const bflc::DropoutArgs drop = dropout_args(dropout_p, seed, step, step_add, site, q, "attention");
    check(bflc::attention_fwd_sm100(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr<float>(),
                                    B, S, H, D, q.stride(0), (float)scale, st(), optp<const int32_t>(lengths), &drop,
                                    causal),
          "attention_fwd_sm100");
  }, py::arg("q"), py::arg("k"), py::arg("v"), py::arg("o"), py::arg("lse"), py::arg("B"), py::arg("S"), py::arg("H"),
     py::arg("scale"), py::arg("lengths") = py::none(), py::arg("dropout_p") = 0.0, py::arg("seed") = 0,
     py::arg("step") = py::none(), py::arg("step_add") = 0, py::arg("site") = 0, py::arg("causal") = false);
  // delta (optional): fp32 workspace of B*H*S floats, required unless (S == 128, no lengths)
  m.def("attention_bwd", [](at::Tensor q, at::Tensor k, at::Tensor v, at::Tensor o, at::Tensor dout, at::Tensor lse,
                            at::Tensor dq, at::Tensor dk, at::Tensor dv, int B, int S, int H, double scale,
                            const OptT& delta, const OptT& lengths, double dropout_p, uint64_t seed,
                            const OptT& step, int64_t step_add, int64_t site, bool causal) {
    const int D = (int)q.size(1) / H;
    const int64_t ld = q.stride(0);
    for (const at::Tensor* t : {&k, &v, &o, &dout, &dq, &dk, &dv})
      TORCH_CHECK(t->stride(1) == 1 && t->stride(0) == ld, "attention: all operands must share one row pitch");
    check_lengths(lengths, q, B);
    if (delta.has_value())
      TORCH_CHECK(delta->scalar_type() == at::kFloat && delta->is_contiguous() &&
                      delta->numel() >= (int64_t)B * H * S && delta->device() == q.device(),
                  "attention: delta must be a contiguous fp32 tensor of B*H*S elements on q's device");
    const bflc::DropoutArgs drop = dropout_args(dropout_p, seed, step, step_add, site, q, "attention");
    check(bflc::attention_bwd_sm100(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), dout.data_ptr(),
                                    lse.data_ptr<float>(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, S, H, D,
                                    ld, (float)scale, st(), optp<float>(delta), optp<const int32_t>(lengths), &drop,
                                    causal),
          "attention_bwd_sm100");
  }, py::arg("q"), py::arg("k"), py::arg("v"), py::arg("o"), py::arg("dout"), py::arg("lse"), py::arg("dq"),
     py::arg("dk"), py::arg("dv"), py::arg("B"), py::arg("S"), py::arg("H"), py::arg("scale"),
     py::arg("delta") = py::none(), py::arg("lengths") = py::none(), py::arg("dropout_p") = 0.0, py::arg("seed") = 0,
     py::arg("step") = py::none(), py::arg("step_add") = 0, py::arg("site") = 0, py::arg("causal") = false);
  // Packed variable-length attention: q, k, v, o and the gradients are [T, H*64] bf16 with one row
  // pitch, sequence b is rows [cu_seqlens[b], cu_seqlens[b+1]); lse and delta are fp32 workspaces of
  // B*H*S_pad floats, S_pad = max_seqlen rounded up to 64.
  m.def("attention_packed_fwd", [](at::Tensor q, at::Tensor k, at::Tensor v, at::Tensor o, at::Tensor lse,
                                   at::Tensor cu_seqlens, int64_t max_seqlen, int H, double scale, double dropout_p,
                                   uint64_t seed, const OptT& step, int64_t step_add, int64_t site) {
    TORCH_CHECK(H > 0 && q.dim() == 2 && q.size(1) % H == 0 && q.size(1) / H == 64,
                "attention_packed: head dim must be 64");
    const int64_t ld = q.stride(0);
    for (const at::Tensor* t : {&q, &k, &v, &o})
      TORCH_CHECK(t->dim() == 2 && t->size(0) == q.size(0) && t->size(1) == q.size(1) && t->stride(1) == 1 &&
                      t->stride(0) == ld,
                  "attention_packed: q, k, v, o must be [T, H*64] with one row pitch");
    const int64_t S_pad = check_packed(cu_seqlens, q, max_seqlen);
    const int B = (int)cu_seqlens.numel() - 1;
    check_workspace(lse, q, (int64_t)B * H * S_pad, "lse");
    const bflc::DropoutArgs drop = dropout_args(dropout_p, seed, step, step_add, site, q, "attention_packed");
    check(bflc::attention_packed_fwd_sm100(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(),
                                           lse.data_ptr<float>(), cu_seqlens.data_ptr<int32_t>(), B,
                                           (int)q.size(0), (int)max_seqlen, H, 64, ld, (float)scale, st(), &drop),
          "attention_packed_fwd_sm100");
  }, py::arg("q"), py::arg("k"), py::arg("v"), py::arg("o"), py::arg("lse"), py::arg("cu_seqlens"),
     py::arg("max_seqlen"), py::arg("H"), py::arg("scale"), py::arg("dropout_p") = 0.0, py::arg("seed") = 0,
     py::arg("step") = py::none(), py::arg("step_add") = 0, py::arg("site") = 0);
  m.def("attention_packed_bwd", [](at::Tensor q, at::Tensor k, at::Tensor v, at::Tensor o, at::Tensor dout,
                                   at::Tensor lse, at::Tensor dq, at::Tensor dk, at::Tensor dv, at::Tensor delta,
                                   at::Tensor cu_seqlens, int64_t max_seqlen, int H, double scale, double dropout_p,
                                   uint64_t seed, const OptT& step, int64_t step_add, int64_t site) {
    TORCH_CHECK(H > 0 && q.dim() == 2 && q.size(1) % H == 0 && q.size(1) / H == 64,
                "attention_packed: head dim must be 64");
    const int64_t ld = q.stride(0);
    for (const at::Tensor* t : {&q, &k, &v, &o, &dout, &dq, &dk, &dv})
      TORCH_CHECK(t->dim() == 2 && t->size(0) == q.size(0) && t->size(1) == q.size(1) && t->stride(1) == 1 &&
                      t->stride(0) == ld,
                  "attention_packed: all operands must be [T, H*64] with one row pitch");
    const int64_t S_pad = check_packed(cu_seqlens, q, max_seqlen);
    const int B = (int)cu_seqlens.numel() - 1;
    check_workspace(lse, q, (int64_t)B * H * S_pad, "lse");
    check_workspace(delta, q, (int64_t)B * H * S_pad, "delta");
    const bflc::DropoutArgs drop = dropout_args(dropout_p, seed, step, step_add, site, q, "attention_packed");
    check(bflc::attention_packed_bwd_sm100(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), dout.data_ptr(),
                                           lse.data_ptr<float>(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(),
                                           cu_seqlens.data_ptr<int32_t>(), B, (int)q.size(0), (int)max_seqlen, H,
                                           64, ld, (float)scale, st(), delta.data_ptr<float>(), &drop),
          "attention_packed_bwd_sm100");
  }, py::arg("q"), py::arg("k"), py::arg("v"), py::arg("o"), py::arg("dout"), py::arg("lse"), py::arg("dq"),
     py::arg("dk"), py::arg("dv"), py::arg("delta"), py::arg("cu_seqlens"), py::arg("max_seqlen"), py::arg("H"),
     py::arg("scale"), py::arg("dropout_p") = 0.0, py::arg("seed") = 0, py::arg("step") = py::none(),
     py::arg("step_add") = 0, py::arg("site") = 0);
  // Hidden dropout: y = (x +) z * keep / (1 - p) over [rows, C] bf16.  Row coordinates: (r / S, r % S),
  // or (seq_ids[r], pos_ids[r]) when seq_ids is given (packed sequences).
  m.def("dropout_add", [](const OptT& x, at::Tensor z, at::Tensor y, int64_t S, const OptT& seq_ids,
                          const OptT& pos_ids, double p, uint64_t seed, const OptT& step, int64_t step_add,
                          int64_t site) {
    TORCH_CHECK(p > 0.0, "dropout_add: dropout_p must be > 0 (p = 0 is the identity)");
    TORCH_CHECK(z.dim() == 2 && z.scalar_type() == at::kBFloat16 && z.is_contiguous() && z.size(1) % 8 == 0,
                "dropout_add: z must be a contiguous bf16 [rows, C] tensor with C % 8 == 0");
    if (x.has_value())
      TORCH_CHECK(x->sizes() == z.sizes() && x->scalar_type() == at::kBFloat16 && x->is_contiguous() &&
                      x->device() == z.device(),
                  "dropout_add: x must be a contiguous bf16 tensor shaped like z");
    TORCH_CHECK(y.sizes() == z.sizes() && y.scalar_type() == at::kBFloat16 && y.is_contiguous() &&
                    y.device() == z.device(),
                "dropout_add: y must be a contiguous bf16 tensor shaped like z");
    const int64_t rows = z.size(0);
    TORCH_CHECK(seq_ids.has_value() == pos_ids.has_value(), "dropout_add: seq_ids and pos_ids go together");
    if (seq_ids.has_value()) {
      for (const OptT* t : {&seq_ids, &pos_ids})
        TORCH_CHECK((*t)->scalar_type() == at::kInt && (*t)->is_contiguous() && (*t)->numel() == rows &&
                        (*t)->device() == z.device(),
                    "dropout_add: seq_ids / pos_ids must be contiguous int32 tensors of one entry per row");
    } else {
      TORCH_CHECK(S > 0, "dropout_add: S (positions per sequence) must be > 0 without seq_ids");
    }
    const bflc::DropoutArgs drop = dropout_args(p, seed, step, step_add, site, z, "dropout_add");
    check(bflc::dropout_add_bf16(x.has_value() ? x->data_ptr() : nullptr, z.data_ptr(), y.data_ptr(), rows,
                                 (int)z.size(1), (int)S, optp<const int32_t>(seq_ids), optp<const int32_t>(pos_ids),
                                 drop, st()),
          "dropout_add_bf16");
  }, py::arg("x"), py::arg("z"), py::arg("y"), py::arg("S"), py::arg("seq_ids"), py::arg("pos_ids"), py::arg("p"),
     py::arg("seed"), py::arg("step"), py::arg("step_add"), py::arg("site"));
  // keep mask of attention dropout, uint8 [B*H, S, S] (a test reference: the same device keep function)
  m.def("dropout_keep_mask", [](at::Tensor mask, int B, int H, int S, double p, uint64_t seed, const OptT& step,
                                int64_t step_add, int64_t site) {
    TORCH_CHECK(p > 0.0, "dropout_keep_mask: dropout_p must be > 0");
    TORCH_CHECK(B > 0 && H > 0 && S > 0 && S % 8 == 0 && S <= 65536, "dropout_keep_mask: need B, H > 0 and S % 8 == 0");
    TORCH_CHECK(mask.scalar_type() == at::kByte && mask.is_contiguous() && mask.numel() == (int64_t)B * H * S * S,
                "dropout_keep_mask: mask must be a contiguous uint8 tensor of B*H*S*S elements");
    const bflc::DropoutArgs drop = dropout_args(p, seed, step, step_add, site, mask, "dropout_keep_mask");
    check(bflc::dropout_keep_mask(mask.data_ptr<uint8_t>(), B, H, S, drop, st()), "dropout_keep_mask");
  });
  // Vocabulary-wide cross-entropy (xent_rows): logits fp32 [M, ld >= V] (row pitch % 4 == 0), targets
  // int32 [M]; loss fp32 [M], hits int32 [>= 1] (+= #argmax == target), dlogits bf16 [M, ldd >= V]
  // contiguous (pad columns [V, ldd) get 0), each optional.
  m.def("xent_rows", [](at::Tensor logits, int64_t V, at::Tensor targets, const OptT& loss, const OptT& hits,
                        const OptT& dlogits, double grad_scale) {
    TORCH_CHECK(logits.dim() == 2 && logits.scalar_type() == at::kFloat && logits.stride(1) == 1 &&
                    logits.stride(0) % 4 == 0 && V >= 1 && V <= logits.stride(0) && V <= logits.size(1),
                "xent_rows: logits must be fp32 [M, >= V] with unit column stride and a row pitch % 4 == 0");
    const int64_t M = logits.size(0);
    TORCH_CHECK(targets.scalar_type() == at::kInt && targets.is_contiguous() && targets.numel() == M &&
                    targets.device() == logits.device(),
                "xent_rows: targets must be a contiguous int32 tensor of M elements on logits' device");
    if (loss.has_value())
      TORCH_CHECK(loss->scalar_type() == at::kFloat && loss->is_contiguous() && loss->numel() >= M &&
                      loss->device() == logits.device(),
                  "xent_rows: loss must be a contiguous fp32 tensor of at least M elements");
    if (hits.has_value())
      TORCH_CHECK(hits->scalar_type() == at::kInt && hits->numel() >= 1 && hits->device() == logits.device(),
                  "xent_rows: hits must be an int32 tensor on logits' device");
    int64_t ldd = 0;
    if (dlogits.has_value()) {
      TORCH_CHECK(dlogits->scalar_type() == at::kBFloat16 && dlogits->dim() == 2 && dlogits->is_contiguous() &&
                      dlogits->size(0) == M && dlogits->size(1) >= V && dlogits->device() == logits.device(),
                  "xent_rows: dlogits must be a contiguous bf16 [M, ldd >= V] tensor");
      ldd = dlogits->size(1);
    }
    check(bflc::xent_rows(logits.data_ptr<float>(), M, (int)V, logits.stride(0), targets.data_ptr<int32_t>(),
                          optp<float>(loss), optp<int32_t>(hits), dlogits.has_value() ? dlogits->data_ptr() : nullptr,
                          ldd, (float)grad_scale, st()),
          "xent_rows");
  }, py::arg("logits"), py::arg("V"), py::arg("targets"), py::arg("loss") = py::none(), py::arg("hits") = py::none(),
     py::arg("dlogits") = py::none(), py::arg("grad_scale") = 1.0);
  m.def("transpose_0213", [](at::Tensor x, at::Tensor y, int d0, int d1, int d2, int d3) {
    check(bflc::transpose_0213_bf16(x.data_ptr(), y.data_ptr(), d0, d1, d2, d3, st()),
          "transpose_0213");
  });
}
