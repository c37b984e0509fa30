// Bindings for the symmetric heap, the federated hot-path kernels, optimizers and
// elementwise helpers.  (GEMM bindings: torch_bindings.cpp.)
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <cmath>
#include <cstring>
#include <memory>
#include <cuda.h>

#include <optional>

#include "bflc_kernels.h"
#include "consensus_math.hpp"
#include "symm_heap.hpp"

namespace py = pybind11;
using OptT = std::optional<at::Tensor>;

namespace {

void check(cudaError_t e, const char* what) {
  TORCH_CHECK(e == cudaSuccess, "bflc::", what, " failed: ", cudaGetErrorString(e));
}
cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

template <typename T>
T* P(int64_t addr) { return reinterpret_cast<T*>(static_cast<uintptr_t>(addr)); }

// A flat buffer of the optimizer, norm, cast and add kernels.  They move exactly n elements through
// 16-byte (fp32, u8, bf16 data) or 8-byte (the optimizer's bf16 shadow) vector accesses and check no
// bounds of their own, so a short, misaligned, strided or mistyped tensor would be read or written
// out of bounds, or silently reinterpreted.
void check_flat(const at::Tensor& t, const char* what, at::ScalarType dtype, int64_t n, int align) {
  TORCH_CHECK(t.is_cuda() && t.is_contiguous() && t.scalar_type() == dtype, what, " must be a contiguous CUDA ",
              c10::toString(dtype), " tensor");
  TORCH_CHECK(t.numel() == n, what, " has ", t.numel(), " elements, expected ", n);
  TORCH_CHECK(reinterpret_cast<uintptr_t>(t.data_ptr()) % align == 0, what, " must be ", align, "-byte aligned");
}

// FedProx arguments: mu must be a finite fp32 >= 0; mu > 0 needs an anchor shaped like master (fp32, n
// elements, 16-byte aligned, master's device).  Returns the anchor the kernel gets: null when mu == 0,
// so that the update is the one without the term, bit for bit.
const float* prox_anchor(const OptT& anchor, double mu, const at::Tensor& master, const char* what) {
  const float m32 = static_cast<float>(mu);
  TORCH_CHECK(std::isfinite(m32) && m32 >= 0.f, what, ": prox_mu must be finite and >= 0, got ", mu);
  if (m32 == 0.f) return nullptr;
  TORCH_CHECK(anchor.has_value(), what, ": prox_mu > 0 needs the anchor (the round's global model)");
  check_flat(*anchor, "anchor", at::kFloat, master.numel(), 16);
  TORCH_CHECK(anchor->device() == master.device(), what, ": anchor must be on master's device");
  return anchor->data_ptr<float>();
}

bflc::FedArgs make_fed(const py::dict& d) {
  bflc::FedArgs f;
  std::memset(&f, 0, sizeof(f));
  f.rank = d["rank"].cast<int>();
  f.n_ranks = d["n_ranks"].cast<int>();
  auto bases = d["peer_bases"].cast<std::vector<int64_t>>();
  TORCH_CHECK((int)bases.size() == f.n_ranks && f.n_ranks <= bflc::kMaxRanks, "bad peer table");
  for (int r = 0; r < f.n_ranks; ++r) f.peers.base[r] = P<char>(bases[r]);
  f.peers.mc_base = P<char>(d["mc_base"].cast<int64_t>());
  auto& l = f.lay;
  l.flags_off = d["flags_off"].cast<int64_t>();
  l.state_off = d["state_off"].cast<int64_t>();
  l.plan_off = d["plan_off"].cast<int64_t>();
  l.scores_off = d["scores_off"].cast<int64_t>();
  l.meta_off = d["meta_off"].cast<int64_t>();
  l.work_master_off = d["work_master_off"].cast<int64_t>();
  l.work_shadow_off = d["work_shadow_off"].cast<int64_t>();
  auto um = d["upload_master_off"].cast<std::vector<int64_t>>();
  auto us = d["upload_shadow_off"].cast<std::vector<int64_t>>();
  l.upload_master_off[0] = um.at(0); l.upload_master_off[1] = um.at(1);
  l.upload_shadow_off[0] = us.at(0); l.upload_shadow_off[1] = us.at(1);
  l.global_off = d["global_off"].cast<int64_t>();
  l.global_shadow_off = d["global_shadow_off"].cast<int64_t>();
  l.ring_off = d["ring_off"].cast<int64_t>();
  l.n_params = d["n_params"].cast<int64_t>();
  l.admit_off = d["admit_off"].cast<int64_t>();
  l.ring_slots = d["ring_slots"].cast<int>();
  return f;
}

struct PyHeap {
  std::unique_ptr<bflc::SymmHeap> h;
};

}  // namespace

void bind_extra(py::module_& m) {
  // ------------------------------------------------------------ symmetric heap
  py::class_<PyHeap>(m, "SymmHeap")
      .def(py::init([](int64_t bytes, int rank, int world, int device, const std::string& mode) {
        bflc::SymmHeap::Mode md = mode == "vmm"   ? bflc::SymmHeap::Mode::VMM
                                  : mode == "ipc" ? bflc::SymmHeap::Mode::IPC
                                                  : bflc::SymmHeap::Mode::LOCAL;
        auto p = std::make_unique<PyHeap>();
        p->h = std::make_unique<bflc::SymmHeap>((size_t)bytes, rank, world, device, md);
        return p;
      }))
      .def("export_handle", [](PyHeap& s) { return py::bytes(s.h->export_handle()); })
      .def("import_handles",
           [](PyHeap& s, const std::vector<py::bytes>& blobs) {
             std::vector<std::string> v;
             for (auto& b : blobs) v.emplace_back(static_cast<std::string>(b));
             s.h->import_handles(v);
           })
      .def("fd_listen", [](PyHeap& s, const std::string& tag) { return s.h->fd_listen(tag); })
      .def("import_via_sockets",
           [](PyHeap& s, const std::vector<std::string>& names) { s.h->import_via_sockets(names); })
      .def("mc_import_via_sockets",
           [](PyHeap& s, const std::vector<std::string>& names) { return s.h->mc_import_via_sockets(names); })
      .def("mc_create_and_export", [](PyHeap& s) { return py::bytes(s.h->mc_create_and_export()); })
      .def("mc_import_and_add",
           [](PyHeap& s, const py::bytes& b) { return s.h->mc_import_and_add(std::string(b)); })
      .def("mc_bind_and_map", [](PyHeap& s) { return s.h->mc_bind_and_map(); })
      .def("local_ptr", [](PyHeap& s) { return reinterpret_cast<int64_t>(s.h->local_ptr()); })
      .def("peer_ptr", [](PyHeap& s, int r) { return reinterpret_cast<int64_t>(s.h->peer_ptr(r)); })
      .def("mc_ptr", [](PyHeap& s) { return reinterpret_cast<int64_t>(s.h->mc_ptr()); })
      .def("bytes", [](PyHeap& s) { return (int64_t)s.h->bytes(); })
      .def("last_error", [](PyHeap& s) { return s.h->last_error(); })
      .def_static("multicast_supported", [](int dev) { return bflc::SymmHeap::multicast_supported(dev); });

  // A torch tensor aliasing raw device memory (heap regions, peer-mapped regions).
  m.def("tensor_from_ptr", [](int64_t ptr, std::vector<int64_t> shape, py::object dtype, int device) {
    auto st = torch::python::detail::py_object_to_dtype(dtype);
    auto opts = at::TensorOptions().dtype(st).device(at::kCUDA, device);
    // target_device: a peer-mapped (VMM / IPC) pointer reports the OWNING GPU as its device;
    // the view must still be a tensor of the local device so local kernels accept it.
    return at::for_blob(P<void>(ptr), shape)
        .deleter([](void*) {})
        .options(opts)
        .target_device(at::Device(at::kCUDA, static_cast<c10::DeviceIndex>(device)))
        .make_tensor();
  });

  m.def("struct_sizes", [] {
    py::dict d;
    d["RoundState"] = sizeof(bflc::RoundState);
    d["RoundPlan"] = sizeof(bflc::RoundPlan);
    d["BlockRecord"] = sizeof(bflc::BlockRecord);
    d["UploadMeta"] = sizeof(bflc::UploadMeta);
    d["AdmitPage"] = sizeof(bflc::AdmitPage);
    d["DpPage"] = sizeof(bflc::DpPage);
    d["dp_norm_off"] = offsetof(bflc::DpPage, norm);
    d["dp_scale_off"] = offsetof(bflc::DpPage, scale);
    d["dp_sigma_off"] = offsetof(bflc::DpPage, sigma);
    d["dp_epoch_off"] = offsetof(bflc::DpPage, epoch);
    d["DpAdapt"] = sizeof(bflc::DpAdapt);
    d["DpClipRecord"] = sizeof(bflc::DpClipRecord);
    d["FLAG_NORM"] = (int)bflc::FLAG_NORM;
    d["GemmDynamic"] = sizeof(bflc::GemmDynamic);
    d["FLAG_COUNT"] = (int)bflc::FLAG_COUNT;
    d["kMaxRanks"] = bflc::kMaxRanks;
    d["kMirrorSeqWord"] = bflc::kMirrorSeqWord;
    d["plan_dyn_off"] = offsetof(bflc::RoundPlan, dyn);
    d["plan_correct_off"] = offsetof(bflc::RoundPlan, correct);
    d["plan_loss_sum_off"] = offsetof(bflc::RoundPlan, loss_sum);
    d["plan_train_correct_off"] = offsetof(bflc::RoundPlan, train_correct);
    d["plan_opt_step_off"] = offsetof(bflc::RoundPlan, opt_step);
    d["plan_is_trainer_off"] = offsetof(bflc::RoundPlan, is_trainer);
    d["plan_is_comm_off"] = offsetof(bflc::RoundPlan, is_comm);
    d["plan_step_barrier_off"] = offsetof(bflc::RoundPlan, step_barrier);
    d["plan_stamps_off"] = offsetof(bflc::RoundPlan, t_stamp);
    d["plan_round_seq_off"] = offsetof(bflc::RoundPlan, round_seq);
    d["plan_opt_total_off"] = offsetof(bflc::RoundPlan, opt_total);
    d["plan_cand_blob_off"] = offsetof(bflc::RoundPlan, cand_blob);
    d["plan_n_cand_off"] = offsetof(bflc::RoundPlan, n_cand);
    d["plan_cand_rank_off"] = offsetof(bflc::RoundPlan, cand_rank);
    d["plan_parity_off"] = offsetof(bflc::RoundPlan, parity);
    d["plan_digest_acc_off"] = offsetof(bflc::RoundPlan, digest_acc);
    d["plan_upload_blocks_off"] = offsetof(bflc::RoundPlan, upload_blocks_done);
    d["plan_consensus_blocks_off"] = offsetof(bflc::RoundPlan, consensus_blocks_done);
    d["dyn_map_index_off"] = offsetof(bflc::GemmDynamic, map_index);
    d["dyn_bias_off"] = offsetof(bflc::GemmDynamic, bias);
    d["dyn_wait_flag_off"] = offsetof(bflc::GemmDynamic, wait_flag);
    d["dyn_wait_value_off"] = offsetof(bflc::GemmDynamic, wait_value);
    d["admit_slot_off"] = offsetof(bflc::AdmitPage, slot);
    d["rec_role_before_off"] = offsetof(bflc::BlockRecord, role_before);
    d["rec_score_rows_off"] = offsetof(bflc::BlockRecord, score_rows);
    d["rec_scored_mask_off"] = offsetof(bflc::BlockRecord, scored_mask);
    d["rec_median_off"] = offsetof(bflc::BlockRecord, median);
    d["rec_n_samples_off"] = offsetof(bflc::BlockRecord, n_samples);
    d["rec_avg_cost_off"] = offsetof(bflc::BlockRecord, avg_cost);
    d["rec_weight_off"] = offsetof(bflc::BlockRecord, weight);
    d["rec_admitted_mask_off"] = offsetof(bflc::BlockRecord, admitted_mask);
    d["rec_weight_by_score_off"] = offsetof(bflc::BlockRecord, weight_by_score);
    d["rec_model_digest_off"] = offsetof(bflc::BlockRecord, model_digest);
    d["rec_seq_off"] = offsetof(bflc::BlockRecord, seq);
    d["rec_agg_off"] = offsetof(bflc::BlockRecord, agg);
    d["state_epoch_off"] = offsetof(bflc::RoundState, epoch);
    d["state_role_off"] = offsetof(bflc::RoundState, role);
    d["state_global_loss_off"] = offsetof(bflc::RoundState, global_loss);
    d["state_digest_off"] = offsetof(bflc::RoundState, model_digest);
    d["CUtensorMap"] = sizeof(CUtensorMap);
    return d;
  });

  // host-side init of the replicated ledger page
  m.def("state_init_bytes", [](int n_ranks, int n_comm, int n_aggregate, std::vector<int> roles, int n_needed) {
    bflc::RoundState st;
    std::memset(&st, 0, sizeof(st));
    st.epoch = 0; st.n_ranks = n_ranks; st.n_comm = n_comm; st.n_aggregate = n_aggregate;
    st.n_needed = (uint32_t)n_needed;
    for (int r = 0; r < n_ranks && r < bflc::kMaxRanks; ++r) st.role[r] = (uint32_t)roles.at(r);
    return py::bytes(reinterpret_cast<const char*>(&st), sizeof(st));
  }, py::arg("n_ranks"), py::arg("n_comm"), py::arg("n_aggregate"), py::arg("roles"), py::arg("n_needed") = 0);

  // ------------------------------------------------------------ fed kernels
  m.def("fed_plan_round", [](const py::dict& fd, std::vector<std::pair<int64_t, bool>> layers,
                             int steps_per_round, bool staged, int64_t blob_stage_ptr, int64_t blob_bytes,
                             std::vector<int64_t> upq_off, int64_t stage_master_ptr) {
    bflc::FedArgs f = make_fed(fd);
    TORCH_CHECK(stage_master_ptr == 0 || staged, "stage_master_ptr: the fp32 staging slots of staged validation");
    bflc::PlanLayer pl[bflc::kMaxPlanLayers];
    TORCH_CHECK((int)layers.size() <= bflc::kMaxPlanLayers, "too many plan layers");
    for (size_t i = 0; i < layers.size(); ++i) {
      pl[i].bias_off = layers[i].first;
      pl[i].use_bias = layers[i].second ? 1 : 0;
    }
    bflc::PlanBlobs pb;
    const bool blobs = blob_bytes > 0;
    if (blobs) {
      TORCH_CHECK(upq_off.size() == 2, "upq_off: heap offsets of the two parity upload blobs");
      pb.stage = P<uint8_t>(blob_stage_ptr); pb.bytes = blob_bytes;
      pb.upq_off[0] = upq_off[0]; pb.upq_off[1] = upq_off[1];
    }
    check(bflc::fed_plan_round(f, pl, (int)layers.size(), steps_per_round, staged ? 1 : 0, cur_stream(),
                               blobs ? &pb : nullptr, P<const float>(stage_master_ptr)),
          "fed_plan_round");
  }, py::arg("fed"), py::arg("layers"), py::arg("steps_per_round"), py::arg("staged"),
     py::arg("blob_stage_ptr") = 0, py::arg("blob_bytes") = 0, py::arg("upq_off") = std::vector<int64_t>{},
     py::arg("stage_master_ptr") = 0);
  // fp8 MLP committee: read each candidate's blob once, unpack it into slot z -- dequantised W1 / W2
  // into stage_dq[z] (bf16, flat parameter layout: offsets w_offs = {w1, w2}), biases into stage[z]
  m.def("fed_pull_blobs", [](const py::dict& fd, int64_t off0, int64_t off1, at::Tensor stage, at::Tensor stage_dq,
                             int in_dim, int hidden, int n_classes, std::vector<int64_t> w_offs) {
    TORCH_CHECK(stage.dim() == 2 && stage_dq.dim() == 2 && stage.size(0) == stage_dq.size(0) &&
                    stage_dq.scalar_type() == at::kBFloat16 && stage.is_contiguous() && stage_dq.is_contiguous(),
                "stage: u8 [slots, blob_bytes]; stage_dq: bf16 [slots, n_params]");
    TORCH_CHECK(w_offs.size() == 2 && w_offs[0] + (int64_t)hidden * in_dim <= stage_dq.size(1) &&
                    w_offs[1] + (int64_t)n_classes * hidden <= stage_dq.size(1) && w_offs[0] % 8 == 0 &&
                    w_offs[1] % 8 == 0,
                "w_offs: 8-aligned element offsets of W1 and W2 inside a stage_dq row");
    const bflc::Mx8Unpack un = bflc::mx8_unpack_args(in_dim, hidden, n_classes, w_offs[0], w_offs[1]);
    check(bflc::fed_pull_blobs(make_fed(fd), off0, off1, un, stage.data_ptr(), stage.size(1), stage_dq.data_ptr(),
                               stage_dq.size(1), cur_stream()),
          "fed_pull_blobs");
  });
  m.def("fed_upload", [](const py::dict& fd, int n_samples, int n_loss_terms, int byz_mode,
                         double byz_scale, int straggle_us) {
    check(bflc::fed_upload(make_fed(fd), n_samples, n_loss_terms, byz_mode, (float)byz_scale, cur_stream(),
                           straggle_us),
          "fed_upload");
  }, py::arg("fed"), py::arg("n_samples"), py::arg("n_loss_terms"), py::arg("byz_mode"), py::arg("byz_scale"),
     py::arg("straggle_us") = 0);
  // rule: 0 FedAvg, 1 coordinate-wise median, 2 trimmed mean (trim values dropped at each end)
  // server_opt: 0 none, 1 momentum, 2 adam, 3 yogi on the rule's result; server_hp = the six fp32
  // constants (lr, b1, b2, c1, c2, tau); server_m_off / server_v_off = heap byte offsets of this
  // rank's state (HeapLayout regions server_m / server_v)
  // dp_mode: 0 off, 1 clip each selected update to L2 norm dp_clip, 2 also Gaussian noise with
  // multiplier dp_noise (FedAvg only), drawn from dp_seed; dp_off = heap byte offset of the DpPage
  // (HeapLayout region dp), whose norm partials fed_update_norms must have filled right before; dp_mode 3 / 4:
  // 1 / 2 with the adaptive clip, read from the DpAdapt header after the DpPage (dp_adapt_bytes), which
  // also write ring_slots clip records after it: dp_bytes, the size of the dp region, must hold all three
  m.def("fed_consensus_aggregate", [](const py::dict& fd, int n_val, bool weight_by_score,
                                      bool two_shot, bool use_mc, int64_t host_mirror,
                                      int64_t bump_seq, int rule, int trim, int server_opt,
                                      const std::vector<float>& server_hp, int64_t server_m_off,
                                      int64_t server_v_off, int dp_mode, double dp_clip, double dp_noise,
                                      uint64_t dp_seed, int64_t dp_off, int64_t dp_bytes) {
    TORCH_CHECK(bflc::agg_rule_valid(rule, trim), "fed_consensus_aggregate: rule must be 0 (FedAvg), 1 (median) "
                "or 2 (trimmed mean, 1 <= trim <= ", bflc::kMaxTrim, "), got rule ", rule, " trim ", trim);
    TORCH_CHECK(rule == bflc::AGG_FEDAVG || !weight_by_score,
                "fed_consensus_aggregate: weight_by_score needs the FedAvg rule");
    bflc::ServerOptArgs so{};
    so.opt = server_opt;
    if (server_opt != bflc::SOPT_NONE) {
      TORCH_CHECK(server_hp.size() == 6, "fed_consensus_aggregate: server_hp = (lr, b1, b2, c1, c2, tau)");
      so.lr = server_hp[0]; so.b1 = server_hp[1]; so.b2 = server_hp[2];
      so.c1 = server_hp[3]; so.c2 = server_hp[4]; so.tau = server_hp[5];
      so.m_off = server_m_off; so.v_off = server_v_off;
    }
    const char* err = bflc::server_opt_check(so.opt, so.lr, so.b1, so.b2, so.tau);
    TORCH_CHECK(*err == '\0', "fed_consensus_aggregate: ", err);
    TORCH_CHECK(server_opt == bflc::SOPT_NONE ||
                    (server_m_off > 0 && server_m_off % 16 == 0 &&
                     (bflc::server_state_vectors(server_opt) < 2 || (server_v_off > 0 && server_v_off % 16 == 0))),
                "fed_consensus_aggregate: server optimizer state offsets must be positive multiples of 16 "
                "(server_v_off for adam / yogi)");
    bflc::DpArgs dp{};
    dp.mode = dp_mode; dp.clip = (float)dp_clip; dp.noise = (float)dp_noise; dp.seed = dp_seed; dp.off = dp_off;
    const char* dperr = bflc::dp_check(dp.mode, dp.clip, dp.noise, rule);
    TORCH_CHECK(*dperr == '\0', "fed_consensus_aggregate: ", dperr);
    TORCH_CHECK(dp_mode == bflc::DP_OFF || (dp_off > 0 && dp_off % 16 == 0),
                "fed_consensus_aggregate: dp_off must be a positive multiple of 16 (the HeapLayout dp region)");
    if (bflc::dp_adaptive(dp_mode)) {
      const int64_t ring = fd["ring_slots"].cast<int64_t>();
      const int64_t need = (int64_t)sizeof(bflc::DpPage) + (int64_t)sizeof(bflc::DpAdapt) +
                           ring * (int64_t)sizeof(bflc::DpClipRecord);
      TORCH_CHECK(dp_bytes >= need, "fed_consensus_aggregate: dp_mode ", dp_mode, " (adaptive clipping) needs a dp "
                  "region of ", need, " bytes (HeapLayout(dp_adaptive=True)), got dp_bytes ", dp_bytes);
    }
    check(bflc::fed_consensus_aggregate(make_fed(fd), n_val, weight_by_score ? 1 : 0,
                                        two_shot ? 1 : 0, use_mc ? 1 : 0, cur_stream(),
                                        P<uint32_t>(host_mirror), P<uint32_t>(bump_seq), rule, trim, &so, &dp),
          "fed_consensus_aggregate");
  }, py::arg("fed"), py::arg("n_val"), py::arg("weight_by_score"), py::arg("two_shot"),
     py::arg("use_mc"), py::arg("host_mirror") = 0, py::arg("bump_seq") = 0, py::arg("rule") = 0,
     py::arg("trim") = 0, py::arg("server_opt") = 0, py::arg("server_hp") = std::vector<float>{},
     py::arg("server_m_off") = 0, py::arg("server_v_off") = 0, py::arg("dp_mode") = 0, py::arg("dp_clip") = 0.0,
     py::arg("dp_noise") = 0.0, py::arg("dp_seed") = 0, py::arg("dp_off") = 0, py::arg("dp_bytes") = 0);
  // adaptive clipping: the DpAdapt header genesis writes right after every replica's DpPage -- C_0, gamma,
  // eta, sigma_b and z_delta = dp_noise_split(noise, count_noise) (0 without noise)
  m.def("dp_adapt_bytes", [](double clip, double noise, double quantile, double lr, double count_noise) {
    const float c = (float)clip, z = (float)noise, q = (float)quantile, l = (float)lr, sb = (float)count_noise;
    const int mode = bflc::dp_mode_of(c, z);
    const char* err = bflc::dp_check(mode, c, z, bflc::AGG_FEDAVG);
    TORCH_CHECK(*err == '\0', "dp_adapt_bytes: ", err);
    err = bflc::dp_adapt_check(mode, z, q, l, sb);
    TORCH_CHECK(*err == '\0' && q != 0.f, "dp_adapt_bytes: ", *err ? err : "dp_clip_quantile is 0 (a fixed clip)");
    bflc::DpAdapt a;
    std::memset(&a, 0, sizeof(a));
    a.clip = c; a.quantile = q; a.lr = l; a.count_noise = sb;
    a.noise_vec = mode == bflc::DP_NOISE ? bflc::dp_noise_split(z, sb) : 0.f;
    return py::bytes(reinterpret_cast<const char*>(&a), sizeof(a));
  }, py::arg("clip"), py::arg("noise"), py::arg("quantile"), py::arg("lr"), py::arg("count_noise"));
  // DP: this rank's slice of every admitted update's squared norm, pushed into every replica's DpPage
  m.def("fed_update_norms", [](const py::dict& fd, int64_t dp_off) {
    TORCH_CHECK(dp_off > 0 && dp_off % 16 == 0, "fed_update_norms: dp_off must be a positive multiple of 16");
    check(bflc::fed_update_norms(make_fed(fd), dp_off, cur_stream()), "fed_update_norms");
  }, py::arg("fed"), py::arg("dp_off"));
  m.def("fed_pull_candidates", [](const py::dict& fd, at::Tensor stage_shadow, const OptT& stage_master,
                                  const OptT& ranges) {
    // ranges: int64 [n][2] device tensor {first float4, float4 count} -- the fp32 parts to pull
    const long long* rp = ranges.has_value() ? reinterpret_cast<const long long*>(ranges->data_ptr<int64_t>())
                                             : nullptr;
    check(bflc::fed_pull_candidates(make_fed(fd), stage_shadow.data_ptr(),
                                    stage_master.has_value() ? stage_master->data_ptr<float>() : nullptr,
                                    cur_stream(), rp, ranges.has_value() ? (int)ranges->size(0) : 0),
          "fed_pull_candidates");
  }, py::arg("fed"), py::arg("stage_shadow"), py::arg("stage_master"), py::arg("ranges") = py::none());
  m.def("fed_wait_trained", [](const py::dict& fd) {
    check(bflc::fed_wait_trained(make_fed(fd), cur_stream()), "fed_wait_trained");
  });
  m.def("set_predicate", [](int64_t ptr) { bflc::set_predicate(P<const int>(ptr)); });
  m.def("current_predicate_is_null", [] { return bflc::current_predicate() == nullptr; });
  m.def("set_pdl", [](bool on) { bflc::set_pdl(on); });
  m.def("pdl_fallbacks", [] { return bflc::pdl_fallbacks(); });
  m.def("set_debug_times", [](int64_t ptr) { bflc::set_debug_times(P<long long>(ptr)); });
  m.def("p2p_read_probe", [](int64_t src, int64_t dst, int64_t n_vec) {
    check(bflc::p2p_read_probe(P<const float4>(src), P<float4>(dst), n_vec, cur_stream()),
          "p2p_read_probe");
  });
  m.def("mc_store_probe", [](int64_t mc_dst, int64_t src, int64_t n_vec) {
    check(bflc::mc_store_probe(P<float4>(mc_dst), P<const float4>(src), n_vec, cur_stream()),
          "mc_store_probe");
  });

  // ------------------------------------------------------------ optimizers
  // whole local-training pass of the 2-layer MLP in one persistent kernel
  m.def("mx8_mlp_layout", [](int in_dim, int hidden) {
    const bflc::Mx8MlpLayout l = bflc::mx8_mlp_layout(in_dim, hidden);
    py::dict d;
    d["w1q"] = l.w1q; d["w1sf"] = l.w1sf; d["w2q"] = l.w2q; d["w2sf"] = l.w2sf;
    d["b1"] = l.b1; d["b2"] = l.b2; d["total"] = l.total; d["kb1"] = l.kb1; d["kb2"] = l.kb2;
    return d;
  });
  // the launcher's phase-plan decision for these shapes on the current device: a dict of plan, epiopt, grid,
  // bm_w and max_clusters, or None where mlp_round would refuse them (then "error" names why)
  m.def("mlp_round_plan", [](int batch, int in_dim, int hidden, int n_classes, bool fp8, bool dpsgd, bool prox,
                             int plan, int epiopt) {
    bflc::MlpPlanRequest q;
    q.batch = batch; q.in_dim = in_dim; q.hidden = hidden; q.n_classes = n_classes;
    q.ncp = (n_classes + 7) / 8 * 8;   // FlatMLP's dlogits row stride
    q.plan = plan; q.epiopt = epiopt; q.fp8 = fp8; q.dpsgd = dpsgd; q.prox = prox;
    bflc::MlpRoundPlan p;
    const cudaError_t e = bflc::mlp_round_plan(q, &p);
    py::dict d;
    d["ok"] = e == cudaSuccess;
    d["error"] = e == cudaSuccess ? std::string() : std::string(cudaGetErrorName(e));
    d["plan"] = p.plan; d["epiopt"] = p.epiopt; d["grid"] = p.grid; d["bm_w"] = p.bm_w;
    d["max_clusters"] = p.max_clusters;
    return d;
  }, py::arg("batch"), py::arg("in_dim"), py::arg("hidden"), py::arg("n_classes"), py::arg("fp8") = false,
     py::arg("dpsgd") = false, py::arg("prox") = false, py::arg("plan") = -1, py::arg("epiopt") = -1);
  m.def("mlp_round", [](at::Tensor x, at::Tensor labels, at::Tensor master, at::Tensor shadow,
                        at::Tensor grad, std::vector<int64_t> offs, at::Tensor h, at::Tensor dlogits,
                        at::Tensor dh, at::Tensor loss_sum, at::Tensor correct, int64_t barrier_ptr,
                        int batch, int steps, int in_dim, int hidden, int n_classes, double lr,
                        bool adam, const OptT& mm, const OptT& vv, int64_t step_base_ptr,
                        const OptT& dbg, int plan, int epiopt, int64_t x_ready_ptr,
                        int64_t round_seq_ptr, const OptT& x_dq, const OptT& work_q, const OptT& work_dq,
                        const OptT& h_dq, const std::optional<py::dict>& fed,
                        std::vector<int64_t> upq_off, int n_samples, int n_loss_terms, int byz_mode,
                        double byz_scale, int straggle_us, const OptT& anchor, double prox_mu,
                        int64_t epoch_rows, double dpsgd_clip, double dpsgd_sigma, uint64_t dpsgd_seed,
                        const OptT& dpsgd_dropped, const OptT& dpsgd_ws, const OptT& dpsgd_dbg) {
    TORCH_CHECK(offs.size() == 4, "offs = element offsets of w1, b1, w2, b2 in the flat buffer");
    // one local epoch = E whole batches; step s reads batch s mod E, so x, x_dq and the labels must
    // hold E * batch rows however many steps (local epochs) the launch runs
    if (epoch_rows == 0) epoch_rows = (int64_t)steps * batch;
    TORCH_CHECK(batch > 0 && steps > 0 && epoch_rows >= batch && epoch_rows % batch == 0 &&
                    epoch_rows / batch <= steps && epoch_rows <= INT32_MAX,
                "mlp_round: epoch_rows must be a multiple of batch, between batch and steps * batch (got ",
                epoch_rows, " rows, batch ", batch, ", steps ", steps, ")");
    auto rows_of = [&](const at::Tensor& t, const char* name, int64_t width, at::ScalarType dt) {
      TORCH_CHECK(t.is_cuda() && t.scalar_type() == dt && t.is_contiguous(), "mlp_round: ", name,
                  " must be a contiguous CUDA tensor of ", c10::toString(dt));
      TORCH_CHECK(t.numel() >= epoch_rows * width, "mlp_round: ", name, " holds ", t.numel() / width,
                  " rows, one local epoch reads ", epoch_rows);
    };
    rows_of(x, "x", in_dim, at::kBFloat16);
    rows_of(labels, "labels", 1, at::kInt);
    if (x_dq.has_value()) rows_of(*x_dq, "x_dq", in_dim, at::kBFloat16);
    bflc::MlpRoundArgs r;
    r.epoch_rows = (int)epoch_rows;
    r.prox_anchor = prox_anchor(anchor, prox_mu, master, "mlp_round");
    r.prox_mu = static_cast<float>(prox_mu);
    r.batch = batch; r.steps = steps; r.in_dim = in_dim; r.hidden = hidden; r.n_classes = n_classes;
    r.ncp = (int)dlogits.stride(0);
    r.n_params = master.numel();
    r.x = x.data_ptr(); r.labels = labels.data_ptr<int32_t>();
    float* mp = master.data_ptr<float>(); float* gp = grad.data_ptr<float>();
    auto* sp = reinterpret_cast<uint16_t*>(shadow.data_ptr());
    r.master = mp; r.shadow = sp; r.grad = gp;
    r.w1_shadow = sp + offs[0]; r.w2_shadow = sp + offs[2];
    r.b1 = mp + offs[1]; r.b2 = mp + offs[3];
    r.gw1 = gp + offs[0]; r.gb1 = gp + offs[1]; r.gw2 = gp + offs[2]; r.gb2 = gp + offs[3];
    r.h = h.data_ptr(); r.dlogits = dlogits.data_ptr(); r.dh = dh.data_ptr();
    r.loss_sum = loss_sum.data_ptr<float>();
    r.correct = reinterpret_cast<unsigned int*>(correct.data_ptr());
    r.barrier = P<unsigned int>(barrier_ptr);
    r.adam = adam;
    r.adam_m = mm.has_value() ? mm->data_ptr<float>() : nullptr;
    r.adam_v = vv.has_value() ? vv->data_ptr<float>() : nullptr;
    r.lr = (float)lr;
    r.step_base = P<const int>(step_base_ptr);
    r.plan = plan; r.epiopt = epiopt;
    r.x_ready = P<const unsigned int>(x_ready_ptr); r.round_seq = P<const unsigned int>(round_seq_ptr);
    if (dbg.has_value()) {
      TORCH_CHECK(dbg->numel() >= (int64_t)steps * 32 && dbg->element_size() == 8, "dbg: int64 [steps, 32]");
      r.dbg = reinterpret_cast<unsigned long long*>(dbg->data_ptr());
    }
    if (x_dq.has_value()) {
      TORCH_CHECK(work_q.has_value() && work_dq.has_value() && h_dq.has_value(),
                  "fp8 mode needs x_dq, work_q, work_dq, h_dq");
      TORCH_CHECK(x_dq->scalar_type() == at::kBFloat16 && work_dq->scalar_type() == at::kBFloat16 &&
                      h_dq->scalar_type() == at::kBFloat16 &&
                      work_dq->numel() >= (int64_t)hidden * in_dim + 64LL * hidden,
                  "x_dq / h_dq: bf16; work_dq: bf16 [hidden * in_dim + 64 * hidden]");
      r.fp8 = true;
      r.x_dq = x_dq->data_ptr();
      r.work_q = work_q->data_ptr<uint8_t>();
      r.work_dq = reinterpret_cast<uint16_t*>(work_dq->data_ptr());
      r.h_dq = h_dq->data_ptr();
    }
    bflc::FedArgs f;
    if (fed.has_value()) {
      f = make_fed(*fed);
      r.fed = &f;
      if (upq_off.size() == 2) { r.upq_off[0] = upq_off[0]; r.upq_off[1] = upq_off[1]; }
      r.n_samples = n_samples; r.n_loss_terms = n_loss_terms; r.byz_mode = byz_mode; r.byz_scale = (float)byz_scale;
      r.straggle_us = straggle_us;
    }
    // DP-SGD (dpsgd_clip > 0): plan 4 with the optimizer in the epilogue, hidden 256, at most 64 classes
    bflc::MlpDpsgdArgs dp;
    if (dpsgd_clip != 0.0) {
      const float c32 = (float)dpsgd_clip, s32 = (float)dpsgd_sigma;
      TORCH_CHECK(std::isfinite(c32) && c32 > 0.f && std::isfinite(s32) && s32 >= 0.f,
                  "mlp_round: DP-SGD needs a finite clip > 0 and a finite sigma >= 0 (fp32)");
      TORCH_CHECK(hidden == 256 && n_classes >= 57 && n_classes <= 64 && (plan == -1 || plan == 4) && epiopt != 0,
                  "mlp_round: DP-SGD runs in phase plan 4 with the optimizer in the epilogue, hidden 256 and 57..64 "
                  "classes (got hidden ", hidden, ", ", n_classes, " classes, plan ", plan, ", epiopt ", epiopt, ")");
      const int64_t mt = (batch + 63) / 64;
      auto f32 = [&](const OptT& t, int64_t n, const char* name) {
        TORCH_CHECK(t.has_value() && t->is_cuda() && t->scalar_type() == at::kFloat && t->is_contiguous() &&
                        t->device() == master.device() && t->numel() >= n,
                    "mlp_round: DP-SGD ", name, " must be a contiguous fp32 CUDA tensor of at least ", n, " elements");
      };
      TORCH_CHECK(dpsgd_dropped.has_value() && dpsgd_dropped->is_cuda() && dpsgd_dropped->scalar_type() == at::kInt &&
                      dpsgd_dropped->numel() == 1 && dpsgd_dropped->device() == master.device(),
                  "mlp_round: DP-SGD dropped must be an int32 [1] tensor on master's device");
      f32(dpsgd_ws, 2 * mt * (hidden + 64), "bias workspace");
      if (dpsgd_dbg.has_value()) f32(dpsgd_dbg, (int64_t)steps * 5 * batch + master.numel(), "dbg");
      dp.clip = c32; dp.sigma = s32; dp.seed = dpsgd_seed;
      dp.dropped = dpsgd_dropped->data_ptr<int32_t>();
      dp.bias_ws = dpsgd_ws->data_ptr<float>();
      dp.dbg = dpsgd_dbg.has_value() ? dpsgd_dbg->data_ptr<float>() : nullptr;
      r.dpsgd = &dp;
    } else {
      TORCH_CHECK(!dpsgd_dropped.has_value() && !dpsgd_ws.has_value() && !dpsgd_dbg.has_value() && dpsgd_sigma == 0.0,
                  "mlp_round: DP-SGD buffers or sigma without dpsgd_clip");
    }
    check(bflc::mlp_round_sm100(r, cur_stream()), "mlp_round_sm100");
  }, py::arg("x"), py::arg("labels"), py::arg("master"), py::arg("shadow"), py::arg("grad"), py::arg("offs"),
     py::arg("h"), py::arg("dlogits"), py::arg("dh"), py::arg("loss_sum"), py::arg("correct"),
     py::arg("barrier_ptr"), py::arg("batch"), py::arg("steps"), py::arg("in_dim"), py::arg("hidden"),
     py::arg("n_classes"), py::arg("lr"), py::arg("adam"), py::arg("m"), py::arg("v"),
     py::arg("step_base_ptr"), py::arg("dbg"), py::arg("plan"), py::arg("epiopt"), py::arg("x_ready_ptr") = 0,
     py::arg("round_seq_ptr") = 0, py::arg("x_dq") = py::none(), py::arg("work_q") = py::none(),
     py::arg("work_dq") = py::none(), py::arg("h_dq") = py::none(),
     py::arg("fed") = py::none(), py::arg("upq_off") = std::vector<int64_t>{}, py::arg("n_samples") = 0,
     py::arg("n_loss_terms") = 0, py::arg("byz_mode") = 0, py::arg("byz_scale") = 0.0,
     py::arg("straggle_us") = 0, py::arg("anchor") = py::none(), py::arg("prox_mu") = 0.0,
     py::arg("epoch_rows") = 0, py::arg("dpsgd_clip") = 0.0, py::arg("dpsgd_sigma") = 0.0,
     py::arg("dpsgd_seed") = 0, py::arg("dpsgd_dropped") = py::none(), py::arg("dpsgd_ws") = py::none(),
     py::arg("dpsgd_dbg") = py::none());
  // committee validation of every candidate in one launch (fwd1 -> relu -> fwd2 -> argmax)
  m.def("mlp_val", [](at::Tensor x, at::Tensor labels, at::Tensor correct, at::Tensor maps,
                      int64_t dyn1_ptr, int64_t dyn2_ptr, int n_val, int in_dim, int hidden,
                      int n_classes, int max_cand, int64_t cand_blob_ptr) {
    TORCH_CHECK(x.scalar_type() == at::kBFloat16, "x: bf16 (fp8 mode: the dequantised MXFP8 x)");
    bflc::MlpValArgs r;
    r.n_val = n_val; r.in_dim = in_dim; r.hidden = hidden; r.n_classes = n_classes;
    r.max_cand = max_cand;
    r.x = x.data_ptr(); r.ldx = x.stride(0);
    r.maps = reinterpret_cast<const CUtensorMap*>(maps.data_ptr());
    r.dyn1 = P<const bflc::GemmDynamic>(dyn1_ptr);
    r.dyn2 = P<const bflc::GemmDynamic>(dyn2_ptr);
    r.labels = labels.data_ptr<int32_t>();
    r.correct = reinterpret_cast<unsigned int*>(correct.data_ptr());
    if (cand_blob_ptr != 0) {    // fp8: biases from the candidates' blobs
      r.fp8 = true;
      r.cand_blob = P<const uint8_t* const>(cand_blob_ptr);
    }
    check(bflc::mlp_val_sm100(r, cur_stream()), "mlp_val_sm100");
  }, py::arg("x"), py::arg("labels"), py::arg("correct"), py::arg("maps"), py::arg("dyn1_ptr"),
     py::arg("dyn2_ptr"), py::arg("n_val"), py::arg("in_dim"), py::arg("hidden"), py::arg("n_classes"),
     py::arg("max_cand"), py::arg("cand_blob_ptr") = 0);
  m.def("quantize_mlp_blob", [](at::Tensor master, std::vector<int64_t> offs, int in_dim, int hidden,
                                int n_classes, at::Tensor blob, const OptT& dq) {
    TORCH_CHECK(offs.size() == 4, "offs = element offsets of w1, b1, w2, b2");
    TORCH_CHECK(!dq.has_value() || (dq->scalar_type() == at::kBFloat16 &&
                                    dq->numel() >= (int64_t)hidden * in_dim + 64LL * hidden),
                "dq: bf16 [hidden * in_dim + 64 * hidden]");
    check(bflc::quantize_mlp_blob(master.data_ptr<float>(), offs[0], offs[1], offs[2], offs[3], in_dim, hidden,
                                  n_classes, blob.data_ptr<uint8_t>(), cur_stream(),
                                  dq.has_value() ? dq->data_ptr() : nullptr),
          "quantize_mlp_blob");
  }, py::arg("master"), py::arg("offs"), py::arg("in_dim"), py::arg("hidden"), py::arg("n_classes"),
     py::arg("blob"), py::arg("dq") = py::none());
  // e4m3 [R, K] + MXFP8 scale chunks -> the exactly dequantised values, bf16 [R, K]
  m.def("mx8_dequant", [](at::Tensor q, at::Tensor sf, at::Tensor dst) {
    TORCH_CHECK(q.dim() == 2 && q.is_contiguous() && q.element_size() == 1, "q: contiguous e4m3 / u8 [R, K]");
    TORCH_CHECK(dst.sizes() == q.sizes() && dst.is_contiguous() && dst.scalar_type() == at::kBFloat16,
                "dst: contiguous bf16 [R, K]");
    check(bflc::mx8_dequant_bf16(q.data_ptr(), sf.data_ptr<uint8_t>(), (int)q.size(0), (int)q.size(1),
                                 dst.data_ptr(), cur_stream()),
          "mx8_dequant_bf16");
  });
  m.def("optim_step",
        [](bool adam, at::Tensor master, at::Tensor grad, const OptT& shadow, const OptT& mm,
           const OptT& vv, double lr, double wd, double b1, double b2, double eps, int step,
           int64_t step_dev_ptr, int64_t active_ptr, bool zero_grad) {
          const int64_t n = master.numel();
          check_flat(master, "master", at::kFloat, n, 16);
          check_flat(grad, "grad", at::kFloat, n, 16);
          if (shadow.has_value()) check_flat(*shadow, "shadow", at::kBFloat16, n, 8);
          if (adam) {
            TORCH_CHECK(mm.has_value() && vv.has_value(), "adam needs m and v");
            check_flat(*mm, "m", at::kFloat, n, 16);
            check_flat(*vv, "v", at::kFloat, n, 16);
            // t = *step_dev + step; t = 0 makes both bias corrections 1 - beta^0 = 0
            TORCH_CHECK(step >= 1, "adam step must be >= 1 (bias correction 1 - beta^t), got ", step);
          }
          bflc::OptimArgs a;
          a.master = master.data_ptr<float>();
          a.grad = grad.data_ptr<float>();
          a.shadow_bf16 = shadow.has_value() ? shadow->data_ptr() : nullptr;
          a.n = master.numel();
          a.lr = (float)lr; a.weight_decay = (float)wd;
          a.m = mm.has_value() ? mm->data_ptr<float>() : nullptr;
          a.v = vv.has_value() ? vv->data_ptr<float>() : nullptr;
          a.beta1 = (float)b1; a.beta2 = (float)b2; a.eps = (float)eps;
          a.step = step;
          a.step_dev = P<const int>(step_dev_ptr);
          a.active = active_ptr ? P<const int>(active_ptr) : bflc::current_predicate();
          a.zero_grad = zero_grad ? 1 : 0;
          check(adam ? bflc::adam_step(a, cur_stream()) : bflc::sgd_step(a, cur_stream()),
                "optim_step");
        });
  // fine-tuning recipe (ops/optim.py): global gradient norm + clip coefficient, and the update with
  // an lr schedule, clipping and decoupled weight decay under a no-decay mask
  m.def("grad_norm_workspace_bytes", [] { return bflc::kGradNormWorkspaceBytes; });
  m.def("grad_norm",
        [](at::Tensor grad, at::Tensor workspace, at::Tensor norms, int64_t index, double max_norm,
           const OptT& skipped, int64_t active_ptr) {
          auto f32 = [](const at::Tensor& t, const char* what) {
            TORCH_CHECK(t.is_cuda() && t.is_contiguous() && t.scalar_type() == at::kFloat, what,
                        " must be a contiguous CUDA float32 tensor");
          };
          check_flat(grad, "grad", at::kFloat, grad.numel(), 16);
          f32(norms, "norms");
          TORCH_CHECK(grad.numel() > 0, "grad is empty");
          TORCH_CHECK(workspace.is_cuda() && workspace.is_contiguous() && workspace.scalar_type() == at::kByte &&
                          workspace.numel() >= bflc::kGradNormWorkspaceBytes &&
                          reinterpret_cast<uintptr_t>(workspace.data_ptr()) % 8 == 0,
                      "workspace must be an 8-byte aligned contiguous CUDA uint8 tensor of grad_norm_workspace_bytes()");
          TORCH_CHECK(0 <= index && index < norms.numel(), "norm index ", index, " outside norms[", norms.numel(), "]");
          TORCH_CHECK(max_norm > 0, "max_norm must be > 0");
          if (skipped.has_value())
            TORCH_CHECK(skipped->is_cuda() && skipped->scalar_type() == at::kInt && skipped->numel() >= 1,
                        "skipped must be a CUDA int32 tensor");
          check(bflc::grad_norm_f32(grad.data_ptr<float>(), grad.numel(), workspace.data_ptr(),
                                    norms.data_ptr<float>() + index, (float)max_norm,
                                    skipped.has_value() ? skipped->data_ptr<int>() : nullptr,
                                    active_ptr ? P<const int>(active_ptr) : bflc::current_predicate(), cur_stream()),
                "grad_norm");
        },
        py::arg("grad"), py::arg("workspace"), py::arg("norms"), py::arg("index"), py::arg("max_norm"),
        py::arg("skipped") = py::none(), py::arg("active_ptr") = 0);
  m.def("optim_recipe_step",
        [](bool adam, at::Tensor master, at::Tensor grad, const OptT& shadow, const OptT& mm, const OptT& vv,
           double lr, double b1, double b2, double eps, int step, int64_t step_dev_ptr, double decay,
           const OptT& no_decay, int schedule, int warmup, int total, const OptT& clip_workspace,
           int64_t active_ptr, bool zero_grad, const OptT& anchor, double prox_mu) {
          const int64_t n = master.numel();
          check_flat(master, "master", at::kFloat, n, 16);
          check_flat(grad, "grad", at::kFloat, n, 16);
          if (shadow.has_value()) check_flat(*shadow, "shadow", at::kBFloat16, n, 8);
          if (adam) {
            TORCH_CHECK(mm.has_value() && vv.has_value(), "adam needs m and v");
            check_flat(*mm, "m", at::kFloat, n, 16);
            check_flat(*vv, "v", at::kFloat, n, 16);
          }
          const float* anc = prox_anchor(anchor, prox_mu, master, "optim_recipe_step");
          // t = *step_dev + step: Adam's bias corrections need t >= 1, the schedule's s = t - 1 >= 0
          TORCH_CHECK(step >= 1, "step must be >= 1, got ", step);
          TORCH_CHECK(schedule >= bflc::kLrConstant && schedule <= bflc::kLrCosine, "schedule id ", schedule,
                      " outside [0, 2] (constant, linear, cosine)");
          TORCH_CHECK(warmup >= 0 && total >= 0, "warmup and total steps must be >= 0");
          TORCH_CHECK(schedule == bflc::kLrConstant || total > warmup,
                      "a decaying schedule needs total steps > warmup steps");
          TORCH_CHECK(decay >= 0, "weight decay must be >= 0");
          if (no_decay.has_value()) {
            TORCH_CHECK(no_decay->is_cuda() && no_decay->is_contiguous() && no_decay->scalar_type() == at::kInt,
                        "no_decay must be a contiguous CUDA int32 tensor");
            TORCH_CHECK(no_decay->numel() == (n + 255) / 256, "no_decay has ", no_decay->numel(),
                        " words, n = ", n, " needs ", (n + 255) / 256, " (one bit per 8 floats)");
          }
          TORCH_CHECK(decay == 0 || no_decay.has_value(), "weight decay needs the no_decay mask");
          if (clip_workspace.has_value())
            TORCH_CHECK(clip_workspace->is_cuda() && clip_workspace->scalar_type() == at::kByte &&
                            clip_workspace->numel() >= bflc::kGradNormWorkspaceBytes &&
                            reinterpret_cast<uintptr_t>(clip_workspace->data_ptr()) % 8 == 0,
                        "clip_workspace must be grad_norm's CUDA uint8 workspace");
          bflc::RecipeArgs a;
          a.master = master.data_ptr<float>();
          a.grad = grad.data_ptr<float>();
          a.shadow_bf16 = shadow.has_value() ? shadow->data_ptr() : nullptr;
          a.n = n;
          a.lr = (float)lr;
          a.m = adam ? mm->data_ptr<float>() : nullptr;
          a.v = adam ? vv->data_ptr<float>() : nullptr;
          a.beta1 = (float)b1; a.beta2 = (float)b2; a.eps = (float)eps;
          a.step = step;
          a.step_dev = P<const int>(step_dev_ptr);
          a.active = active_ptr ? P<const int>(active_ptr) : bflc::current_predicate();
          a.zero_grad = zero_grad ? 1 : 0;
          a.decay = (float)decay;
          a.no_decay = no_decay.has_value() ? reinterpret_cast<const uint32_t*>(no_decay->data_ptr<int>()) : nullptr;
          a.schedule = schedule; a.warmup = warmup; a.total = total;
          a.clip = clip_workspace.has_value() ? static_cast<const bflc::GradNormState*>(clip_workspace->data_ptr())
                                              : nullptr;
          a.anchor = anc;
          a.mu = static_cast<float>(prox_mu);
          check(adam ? bflc::adam_recipe_step(a, cur_stream()) : bflc::sgd_recipe_step(a, cur_stream()),
                "optim_recipe_step");
        },
        py::arg("adam"), py::arg("master"), py::arg("grad"), py::arg("shadow"), py::arg("m"), py::arg("v"),
        py::arg("lr"), py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("step"), py::arg("step_dev_ptr"),
        py::arg("decay"), py::arg("no_decay"), py::arg("schedule"), py::arg("warmup"), py::arg("total"),
        py::arg("clip_workspace"), py::arg("active_ptr") = 0, py::arg("zero_grad") = true,
        py::arg("anchor") = py::none(), py::arg("prox_mu") = 0.0);

  // ------------------------------------------------------------ elementwise
  m.def("cast_f32_to_bf16", [](at::Tensor src, at::Tensor dst) {
    check_flat(src, "src", at::kFloat, src.numel(), 16);
    check_flat(dst, "dst", at::kBFloat16, src.numel(), 16);
    check(bflc::cast_f32_to_bf16(src.data_ptr<float>(), dst.data_ptr(), src.numel(), cur_stream()),
          "cast_f32_to_bf16");
  });
  m.def("cast_bf16_to_f32", [](at::Tensor src, at::Tensor dst) {
    check(bflc::cast_bf16_to_f32(src.data_ptr(), dst.data_ptr<float>(), src.numel(), cur_stream()),
          "cast_bf16_to_f32");
  });
  // input preparation: u8 pixels -> bf16 (+ e4m3 and MXFP8 scale chunks); the chunked variant is
  // the flag-driven side-branch kernel of the host->device input pipeline (see k_prep_chunks)
  m.def("prep_inputs", [](at::Tensor src, const OptT& dst_bf16, const OptT& dst_q, const OptT& dst_sf,
                          double scale, const OptT& dst_dq) {
    TORCH_CHECK(src.dim() == 2 && src.is_contiguous(), "src: contiguous u8 [R, K]");
    TORCH_CHECK(!dst_dq.has_value() || (dst_dq->scalar_type() == at::kBFloat16 && dst_dq->numel() >= src.numel()),
                "dst_dq: bf16 [R, K]");
    check(bflc::prep_inputs_u8(src.data_ptr<uint8_t>(), dst_bf16.has_value() ? dst_bf16->data_ptr() : nullptr,
                               dst_q.has_value() ? dst_q->data_ptr() : nullptr,
                               dst_sf.has_value() ? dst_sf->data_ptr<uint8_t>() : nullptr, (int)src.size(0),
                               (int)src.size(1), (float)scale, cur_stream(),
                               dst_dq.has_value() ? dst_dq->data_ptr() : nullptr),
          "prep_inputs_u8");
  }, py::arg("src"), py::arg("dst_bf16"), py::arg("dst_q"), py::arg("dst_sf"), py::arg("scale"),
     py::arg("dst_dq") = py::none());
  m.def("prep_inputs_chunks", [](at::Tensor src, const OptT& dst_bf16, const OptT& dst_q, const OptT& dst_sf,
                                 int rows_per_chunk, int n_chunks, double scale, at::Tensor in_flags,
                                 at::Tensor in_seq, at::Tensor cnt, at::Tensor ready, at::Tensor err,
                                 const OptT& dst_dq) {
    TORCH_CHECK(src.dim() == 2 && src.is_contiguous() && src.scalar_type() == at::kByte, "src: contiguous u8 [R, K]");
    TORCH_CHECK(rows_per_chunk > 0 && n_chunks > 0, "prep_inputs_chunks: rows_per_chunk and n_chunks must be > 0");
    // the kernel converts rows [0, rows_per_chunk * n_chunks) and keeps one flag word per chunk
    const int64_t R = (int64_t)rows_per_chunk * n_chunks, K = src.size(1);
    TORCH_CHECK(src.size(0) >= R, "prep_inputs_chunks: src holds ", src.size(0), " rows, ", n_chunks,
                " chunks of ", rows_per_chunk, " need ", R);
    auto dst = [&](const OptT& t, const char* name, at::ScalarType dt, int64_t n) {
      TORCH_CHECK(!t.has_value() || (t->scalar_type() == dt && t->is_contiguous() && t->numel() >= n),
                  "prep_inputs_chunks: ", name, " must be contiguous ", c10::toString(dt), " of at least ", n,
                  " elements");
    };
    dst(dst_bf16, "dst_bf16", at::kBFloat16, R * K);
    dst(dst_dq, "dst_dq", at::kBFloat16, R * K);
    dst(dst_q, "dst_q", at::kByte, R * K);
    dst(dst_sf, "dst_sf", at::kByte, (R + 127) / 128 * ((K + 127) / 128) * 512);
    for (const at::Tensor* t : {&in_flags, &cnt, &ready})
      TORCH_CHECK(t->is_contiguous() && t->element_size() == 4 && t->numel() >= n_chunks,
                  "prep_inputs_chunks: in_flags, cnt and ready need one 32-bit word per chunk (", n_chunks, ")");
    TORCH_CHECK(in_seq.element_size() == 4 && in_seq.numel() >= 1 && err.element_size() == 4 && err.numel() >= 1,
                "prep_inputs_chunks: in_seq and err are 32-bit words");
    check(bflc::prep_inputs_u8_chunks(src.data_ptr<uint8_t>(), dst_bf16.has_value() ? dst_bf16->data_ptr() : nullptr,
                                      dst_q.has_value() ? dst_q->data_ptr() : nullptr,
                                      dst_sf.has_value() ? dst_sf->data_ptr<uint8_t>() : nullptr, rows_per_chunk,
                                      (int)src.size(1), n_chunks, (float)scale, in_flags.data_ptr<int32_t>(),
                                      in_seq.data_ptr<int32_t>(), reinterpret_cast<unsigned int*>(cnt.data_ptr()),
                                      reinterpret_cast<unsigned int*>(ready.data_ptr()),
                                      reinterpret_cast<unsigned int*>(err.data_ptr()), cur_stream(),
                                      dst_dq.has_value() ? dst_dq->data_ptr() : nullptr),
          "prep_inputs_u8_chunks");
  }, py::arg("src"), py::arg("dst_bf16"), py::arg("dst_q"), py::arg("dst_sf"), py::arg("rows_per_chunk"),
     py::arg("n_chunks"), py::arg("scale"), py::arg("in_flags"), py::arg("in_seq"), py::arg("cnt"),
     py::arg("ready"), py::arg("err"), py::arg("dst_dq") = py::none());
  // cudaGraphLaunch of an instantiated graph (torch.cuda.CUDAGraph.raw_cuda_graph_exec()) on a
  // given stream: the per-round launch without the stream-guard / generator bookkeeping of
  // CUDAGraph.replay() on the Python path.
  m.def("graph_launch", [](int64_t exec_ptr, int64_t stream_ptr) {
    check(cudaGraphLaunch(reinterpret_cast<cudaGraphExec_t>(static_cast<uintptr_t>(exec_ptr)),
                          reinterpret_cast<cudaStream_t>(static_cast<uintptr_t>(stream_ptr))),
          "cudaGraphLaunch");
  });
  m.def("h2d_pipeline", [](int64_t host_x, int64_t dev_x, int64_t chunk_bytes, int c_begin, int c_end,
                           int64_t host_y, int64_t dev_y, int64_t y_bytes, int64_t dev_flags,
                           int64_t host_seq, int64_t stream_ptr, bool write_value) {
    // chunks [c_begin, c_end); the labels travel with chunk 0 (y_bytes > 0).  A chunk's tag is a
    // stream-ordered 32-bit write behind its copy: cuStreamWriteValue32 (a stream memory
    // operation, no copy-engine descriptor) or, as a fallback, a 4-byte copy of *host_seq.
    using WriteFn = CUresult (*)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
    static WriteFn wv = [] {
      void* sym = nullptr;
      cudaDriverEntryPointQueryResult q;
      if (cudaGetDriverEntryPoint("cuStreamWriteValue32", &sym, cudaEnableDefault, &q) != cudaSuccess ||
          q != cudaDriverEntryPointSuccess)
        sym = nullptr;
      return reinterpret_cast<WriteFn>(sym);
    }();
    cudaStream_t s = reinterpret_cast<cudaStream_t>(static_cast<uintptr_t>(stream_ptr));
    const uint32_t tag = static_cast<uint32_t>(*P<const int32_t>(host_seq));
    if (y_bytes > 0)
      check(cudaMemcpyAsync(P<void>(dev_y), P<const void>(host_y), (size_t)y_bytes, cudaMemcpyHostToDevice, s),
            "h2d labels");
    for (int c = c_begin; c < c_end; ++c) {
      check(cudaMemcpyAsync(P<char>(dev_x) + c * chunk_bytes, P<const char>(host_x) + c * chunk_bytes,
                            (size_t)chunk_bytes, cudaMemcpyHostToDevice, s), "h2d chunk");
      bool done = false;
      if (write_value && wv != nullptr)
        done = wv(reinterpret_cast<CUstream>(s), static_cast<CUdeviceptr>(dev_flags + 4 * c), tag, 0u) == CUDA_SUCCESS;
      if (!done)
        check(cudaMemcpyAsync(P<int32_t>(dev_flags) + c, P<const void>(host_seq), 4, cudaMemcpyHostToDevice, s),
              "h2d tag");
    }
  }, py::arg("host_x"), py::arg("dev_x"), py::arg("chunk_bytes"), py::arg("c_begin"), py::arg("c_end"),
     py::arg("host_y"), py::arg("dev_y"), py::arg("y_bytes"), py::arg("dev_flags"), py::arg("host_seq"),
     py::arg("stream_ptr"), py::arg("write_value") = true);
  m.def("cast_u8_to_bf16", [](at::Tensor src, at::Tensor dst, double scale) {
    check_flat(src, "src", at::kByte, src.numel(), 16);
    check_flat(dst, "dst", at::kBFloat16, src.numel(), 16);
    check(bflc::cast_u8_to_bf16(src.data_ptr<uint8_t>(), dst.data_ptr(), src.numel(), (float)scale,
                                cur_stream()),
          "cast_u8_to_bf16");
  });
  m.def("quantize_fp8", [](at::Tensor src, at::Tensor dst, double inv_scale) {
    check(bflc::quantize_fp8(src.data_ptr(), reinterpret_cast<uint8_t*>(dst.data_ptr()),
                             src.numel(), (float)inv_scale, cur_stream()),
          "quantize_fp8");
  });
  m.def("amax_bf16", [](at::Tensor src, at::Tensor out) {
    check(bflc::amax_bf16(src.data_ptr(), src.numel(), out.data_ptr<float>(), cur_stream()),
          "amax_bf16");
  });
  m.def("fill_f32", [](at::Tensor dst, double v) {
    check(bflc::fill_f32(dst.data_ptr<float>(), dst.numel(), (float)v, cur_stream()), "fill_f32");
  });
  m.def("add_bf16", [](at::Tensor a, at::Tensor b, at::Tensor out) {
    check_flat(a, "a", at::kBFloat16, a.numel(), 16);
    check_flat(b, "b", at::kBFloat16, a.numel(), 16);
    check_flat(out, "out", at::kBFloat16, a.numel(), 16);
    check(bflc::add_bf16(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.numel(), cur_stream()),
          "add_bf16");
  });
}
