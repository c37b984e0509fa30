// pybind11 module `_ledger`: the C++ ledger runtime without any CUDA / torch dependency,
// so the protocol tests and the gloo plumbing path run on a CPU-only box.
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <cstring>

#include "consensus_math.hpp"
#include "ledger.hpp"

namespace py = pybind11;
using namespace bflc;

namespace {
py::bytes h2b(const Hash256& h) { return py::bytes(reinterpret_cast<const char*>(h.data()), 32); }

py::dict block_to_dict(const Block& b) {
  py::dict d;
  d["index"] = b.index; d["epoch"] = b.epoch;
  d["prev_hash"] = hex(b.prev_hash); d["hash"] = hex(b.hash);
  d["role_before"] = b.role_before; d["role_after"] = b.role_after;
  d["admitted"] = b.admitted; d["committee"] = b.committee; d["scores"] = b.scores;
  d["median"] = b.median; d["selected"] = b.selected; d["weight"] = b.weight;
  d["global_loss"] = b.global_loss; d["model_hash"] = hex(b.model_hash);
  d["device_digest"] = b.device_digest; d["from_device"] = (bool)b.from_device;
  return d;
}

std::vector<float> arr_to_vec(const py::array_t<float, py::array::c_style | py::array::forcecast>& a) {
  return std::vector<float>(a.data(), a.data() + a.size());
}
}  // namespace

PYBIND11_MODULE(_ledger, m) {
  m.doc() = "bflc_demo_b200 C++ ledger runtime";
  m.attr("EPOCH_NOT_STARTED") = kEpochNotStarted;
  m.attr("ROLE_TRAINER") = (uint32_t)ROLE_TRAINER;
  m.attr("ROLE_COMM") = (uint32_t)ROLE_COMM;

  py::enum_<Status>(m, "Status")
      .value("OK", Status::OK).value("NOT_STARTED", Status::NOT_STARTED)
      .value("STALE_EPOCH", Status::STALE_EPOCH).value("DUPLICATE", Status::DUPLICATE)
      .value("QUOTA_FULL", Status::QUOTA_FULL).value("NOT_COMMITTEE", Status::NOT_COMMITTEE)
      .value("UNKNOWN_CLIENT", Status::UNKNOWN_CLIENT).value("BAD_PAYLOAD", Status::BAD_PAYLOAD)
      .value("AGGREGATED", Status::AGGREGATED).value("NOT_TRAINER", Status::NOT_TRAINER)
      .value("NOT_READY", Status::NOT_READY);

  py::class_<LedgerConfig>(m, "LedgerConfig")
      .def(py::init<>())
      .def_readwrite("client_num", &LedgerConfig::client_num)
      .def_readwrite("comm_count", &LedgerConfig::comm_count)
      .def_readwrite("aggregate_count", &LedgerConfig::aggregate_count)
      .def_readwrite("needed_update_count", &LedgerConfig::needed_update_count)
      .def_readwrite("learning_rate", &LedgerConfig::learning_rate)
      .def_readwrite("model_size", &LedgerConfig::model_size)
      .def_readwrite("weight_by_score", &LedgerConfig::weight_by_score)
      .def_readwrite("solo", &LedgerConfig::solo)
      .def_readwrite("seed", &LedgerConfig::seed)
      .def_readwrite("aggregation", &LedgerConfig::aggregation)
      .def_readwrite("trim", &LedgerConfig::trim)
      .def_readwrite("server_opt", &LedgerConfig::server_opt)
      .def_readwrite("server_lr", &LedgerConfig::server_lr)
      .def_readwrite("server_beta1", &LedgerConfig::server_beta1)
      .def_readwrite("server_beta2", &LedgerConfig::server_beta2)
      .def_readwrite("server_tau", &LedgerConfig::server_tau)
      .def_readwrite("dp_clip", &LedgerConfig::dp_clip)
      .def_readwrite("dp_noise", &LedgerConfig::dp_noise)
      .def_readwrite("dp_seed", &LedgerConfig::dp_seed)
      .def_readwrite("dp_clip_quantile", &LedgerConfig::dp_clip_quantile)
      .def_readwrite("dp_clip_lr", &LedgerConfig::dp_clip_lr)
      .def_readwrite("dp_count_noise", &LedgerConfig::dp_count_noise)
      .def("dp_adaptive", &LedgerConfig::dp_adaptive)
      .def("dp_kernel_mode", &LedgerConfig::dp_kernel_mode)
      .def("dp_mode", &LedgerConfig::dp_mode)
      .def("validate", &LedgerConfig::validate);

  py::class_<Ledger>(m, "Ledger")
      .def(py::init<const LedgerConfig&>())
      .def("RegisterNode", &Ledger::RegisterNode)
      .def("QueryState", &Ledger::QueryState)
      .def("QueryGlobalModel",
           [](Ledger& L) {
             auto r = L.QueryGlobalModel();
             py::array_t<float> a(r.first.size());
             std::memcpy(a.mutable_data(), r.first.data(), r.first.size() * sizeof(float));
             return py::make_tuple(a, r.second);
           })
      .def("UploadLocalUpdate",
           [](Ledger& L, int client,
              py::array_t<float, py::array::c_style | py::array::forcecast> delta,
              uint32_t n_samples, float avg_cost, int ep) {
             UpdateMeta meta;
             meta.n_samples = n_samples; meta.avg_cost = avg_cost;
             std::vector<float> d = arr_to_vec(delta);
             py::gil_scoped_release rel;
             return L.UploadLocalUpdate(client, d, meta, ep);
           })
      .def("UploadScores",
           [](Ledger& L, int client, int ep, const std::map<int, float>& scores) {
             return L.UploadScores(client, ep, scores);
           })
      .def("QueryAllUpdates",
           [](Ledger& L) {
             py::list out;
             for (auto& u : L.QueryAllUpdates()) {
               py::dict d;
               py::array_t<float> a(u.delta.size());
               std::memcpy(a.mutable_data(), u.delta.data(), u.delta.size() * sizeof(float));
               d["sender"] = u.sender; d["delta"] = a; d["n_samples"] = u.meta.n_samples;
               d["avg_cost"] = u.meta.avg_cost; d["arrival"] = u.arrival;
               out.append(d);
             }
             return out;
           })
      .def("Bootstrap", &Ledger::Bootstrap)
      .def("AppendDeviceRound",
           [](Ledger& L, const py::dict& d) {
             Ledger::DeviceRound r;
             r.epoch = d["epoch"].cast<int>();
             r.role_before = d["role_before"].cast<std::vector<uint32_t>>();
             r.role_after = d["role_after"].cast<std::vector<uint32_t>>();
             r.score_rows = d["score_rows"].cast<std::vector<std::vector<float>>>();
             r.scored_mask = d["scored_mask"].cast<std::vector<uint32_t>>();
             r.n_samples = d["n_samples"].cast<std::vector<uint32_t>>();
             r.avg_cost = d["avg_cost"].cast<std::vector<float>>();
             r.admitted_mask = d["admitted_mask"].cast<uint32_t>();
             r.selected_mask = d["selected_mask"].cast<uint32_t>();
             r.global_loss = d["global_loss"].cast<float>();
             r.model_digest = d["model_digest"].cast<uint64_t>();
             r.weight_by_score = d["weight_by_score"].cast<int>();
             r.agg = d.contains("agg") ? d["agg"].cast<uint32_t>() : 0u;   // absent: a FedAvg record
             if (d.contains("clip")) {   // adaptive clipping: the round's clip record
               r.has_clip = 1;
               r.clip = d["clip"].cast<float>();
               r.count = d["count"].cast<float>();
               r.n_sel = d["n_sel"].cast<uint32_t>();
             }
             return L.AppendDeviceRound(r);
           })
      .def("epoch", &Ledger::epoch)
      .def("roles", &Ledger::roles)
      .def("update_count", &Ledger::update_count)
      .def("score_count", &Ledger::score_count)
      .def("n_blocks", &Ledger::n_blocks)
      .def("last_global_loss", &Ledger::last_global_loss)
      .def("blocks",
           [](Ledger& L) {
             py::list out;
             for (auto& b : L.blocks()) out.append(block_to_dict(b));
             return out;
           })
      .def("counters",
           [](Ledger& L) {
             OpCounters c = L.counters();
             py::dict d;
             d["calls"] = c.calls; d["register_ok"] = c.register_ok; d["uploads_ok"] = c.uploads_ok;
             d["uploads_rejected"] = c.uploads_rejected; d["scores_ok"] = c.scores_ok;
             d["scores_rejected"] = c.scores_rejected; d["aggregations"] = c.aggregations;
             d["queries"] = c.queries;
             return d;
           })
      .def("drain_log", &Ledger::drain_log)
      .def("state_hash", [](Ledger& L) { return hex(L.state_hash()); })
      .def("server_state",
           [](Ledger& L) {   // (m, v) float32 arrays, empty before the first host aggregation
             auto st = L.server_state();
             return py::make_tuple(py::array_t<float>(st.first.size(), st.first.data()),
                                   py::array_t<float>(st.second.size(), st.second.data()));
           })
      .def("dp_clip_now", &Ledger::dp_clip_now)
      .def("last_clip_step",
           [](Ledger& L) {   // (C_t, b~, n_sel) of the last aggregated round (adaptive clipping)
             const Ledger::ClipStep s = L.last_clip_step();
             return py::make_tuple(s.clip, s.count, s.n_sel);
           })
      .def("verify_chain", &Ledger::verify_chain)
      .def("snapshot", [](Ledger& L) { return py::bytes(L.snapshot()); })
      .def_static("restore", [](const py::bytes& b, uint64_t dp_seed) { return Ledger::restore(std::string(b), dp_seed); },
                  py::arg("blob"), py::arg("dp_seed") = 0)
      .def("config", [](Ledger& L) { return L.config(); });

  // ABI-style method table + dispatcher-by-signature (reference C:46-52, C:132-167, C:312-318)
  m.def("method_table", [] {
    int n = 0;
    const MethodInfo* t = method_table(&n);
    py::list out;
    for (int i = 0; i < n; ++i)
      out.append(py::make_tuple((int)t[i].id, std::string(t[i].signature), t[i].is_view));
    return out;
  });
  m.def("method_from_signature", [](const std::string& s) { return (int)method_from_signature(s); });

  m.def("sha256_hex", [](const py::bytes& b) {
    std::string s = b;
    return hex(sha256(s.data(), s.size()));
  });
  m.def("status_name", [](Status s) { return std::string(status_name(s)); });

  m.attr("AGG_FEDAVG") = (int)AGG_FEDAVG;
  m.attr("AGG_MEDIAN") = (int)AGG_MEDIAN;
  m.attr("AGG_TRIMMED_MEAN") = (int)AGG_TRIMMED_MEAN;
  m.def("agg_word", [](int rule, int trim, int server_opt, int dp) { return agg_word(rule, trim, server_opt, dp); },
        py::arg("rule"), py::arg("trim"), py::arg("server_opt") = 0, py::arg("dp") = 0);
  m.attr("DP_OFF") = (int)DP_OFF;
  m.attr("DP_CLIP") = (int)DP_CLIP;
  m.attr("DP_NOISE") = (int)DP_NOISE;
  m.attr("DP_CLIP_ADAPT") = (int)DP_CLIP_ADAPT;
  m.attr("DP_NOISE_ADAPT") = (int)DP_NOISE_ADAPT;
  m.attr("DP_CLIP_SITE") = kDpClipSite;
  m.attr("DP_EXP_MAX") = kDpExpMax;
  // adaptive clipping's shared definitions (consensus_math.hpp), for the host tests
  m.def("dp_exp_values", [](py::array_t<float, py::array::c_style | py::array::forcecast> x) {
    py::array_t<float> out(x.size());
    const float* px = x.data();
    float* po = out.mutable_data();
    for (py::ssize_t i = 0; i < x.size(); ++i) po[i] = dp_exp(px[i]);
    return out;
  });
  m.def("dp_noised_count", [](uint32_t b, int n_sel, float count_noise, uint64_t seed, uint32_t epoch) {
    return dp_noised_count(b, n_sel, count_noise, seed, epoch);
  });
  m.def("dp_clip_next", [](float clip, float count, int n_sel, float quantile, float lr) {
    if (n_sel < 1) throw std::invalid_argument("n_sel must be >= 1");
    return dp_clip_next(clip, count, n_sel, quantile, lr);
  });
  m.def("dp_noise_split", [](float noise, float count_noise) { return dp_noise_split(noise, count_noise); });
  // the DP noise xi_i of coordinates first .. first + n - 1 of round `epoch` (dp_gauss4), float32 [n]
  m.def("dp_gauss_coordinates", [](uint64_t seed, uint32_t epoch, uint64_t first, py::ssize_t n) {
    if (n < 0) throw std::invalid_argument("n must be >= 0");
    py::array_t<float> out(n);
    float* p = out.mutable_data();
    {
      py::gil_scoped_release rel;
      dp_gauss_fill(seed, epoch, first, p, static_cast<size_t>(n));
    }
    return out;
  }, py::arg("seed"), py::arg("epoch"), py::arg("first"), py::arg("n"));
  // Box-Muller of raw 32-bit words (dp_box_muller): a, b uint32 [n] -> (z0, z1) float32 [n]
  m.def("dp_box_muller_words",
        [](const py::array_t<uint32_t, py::array::c_style | py::array::forcecast>& a,
           const py::array_t<uint32_t, py::array::c_style | py::array::forcecast>& b) {
          const py::ssize_t n = a.size();
          if (b.size() != n) throw std::invalid_argument("a, b must have the same size");
          py::array_t<float> z0(n), z1(n);
          const uint32_t *pa = a.data(), *pb = b.data();
          float *p0 = z0.mutable_data(), *p1 = z1.mutable_data();
          for (py::ssize_t i = 0; i < n; ++i) dp_box_muller(pa[i], pb[i], p0[i], p1[i]);
          return py::make_tuple(z0, z1);
        },
        py::arg("a"), py::arg("b"));
  // one update's clip against the global model: g, u float32 [P], clip > 0 -> (v, n, s) with n the
  // norm of u - g (fp64 squares summed in ascending index order), s = dp_scale(n, clip), v = u when
  // s == 1 else g + s * (u - g)
  m.def("dp_clip_coordinates",
        [](const py::array_t<float, py::array::c_style | py::array::forcecast>& g,
           const py::array_t<float, py::array::c_style | py::array::forcecast>& u, float clip) {
          if (!(std::isfinite(clip) && clip > 0.f)) throw std::invalid_argument("clip must be finite and > 0");
          const py::ssize_t p = g.size();
          if (g.ndim() != 1 || u.size() != p) throw std::invalid_argument("g, u must be float32 [P]");
          const float *pg = g.data(), *pu = u.data();
          double sum = 0.0;
          for (py::ssize_t i = 0; i < p; ++i) {
            const double d = so_sub(pu[i], pg[i]);
            sum += d * d;
          }
          const float nrm = dp_norm(sum), s = dp_scale(nrm, clip);
          py::array_t<float> v(p);
          float* pv = v.mutable_data();
          for (py::ssize_t i = 0; i < p; ++i) pv[i] = dp_bits(s) == 0x3F800000u ? pu[i] : dp_clip_value(pg[i], pu[i], s);
          return py::make_tuple(v, nrm, s);
        },
        py::arg("g"), py::arg("u"), py::arg("clip"));
  m.attr("SOPT_NONE") = (int)SOPT_NONE;
  m.attr("SOPT_MOMENTUM") = (int)SOPT_MOMENTUM;
  m.attr("SOPT_ADAM") = (int)SOPT_ADAM;
  m.attr("SOPT_YOGI") = (int)SOPT_YOGI;
  // the six fp32 constants (lr, b1, b2, c1, c2, tau) of server_step for fp32 lr / betas / tau
  m.def("server_opt_params", [](float lr, float b1, float b2, float tau) {
    const ServerOptParams p = server_opt_params(lr, b1, b2, tau);
    return py::make_tuple(p.lr, p.b1, p.b2, p.c1, p.c2, p.tau);
  });
  // server_step over every coordinate: g, a, m, v float32 [P] (v ignored by momentum), opt 1..3,
  // params = (lr, b1, b2, c1, c2, tau) -> (g', m', v')
  m.def("server_step_coordinates",
        [](const py::array_t<float, py::array::c_style | py::array::forcecast>& g,
           const py::array_t<float, py::array::c_style | py::array::forcecast>& a,
           const py::array_t<float, py::array::c_style | py::array::forcecast>& m0,
           const py::array_t<float, py::array::c_style | py::array::forcecast>& v0, int opt,
           const std::vector<float>& params) {
          if (opt < SOPT_MOMENTUM || opt > SOPT_YOGI) throw std::invalid_argument("opt must be 1, 2 or 3");
          if (params.size() != 6) throw std::invalid_argument("params = (lr, b1, b2, c1, c2, tau)");
          const py::ssize_t p = g.size();
          if (g.ndim() != 1 || a.size() != p || m0.size() != p || v0.size() != p)
            throw std::invalid_argument("g, a, m, v must be float32 [P]");
          const ServerOptParams sp{params[0], params[1], params[2], params[3], params[4], params[5]};
          py::array_t<float> go(p), mo(p), vo(p);
          const float *pg = g.data(), *pa = a.data(), *pm = m0.data(), *pv = v0.data();
          float *dg = go.mutable_data(), *dm = mo.mutable_data(), *dv = vo.mutable_data();
          for (py::ssize_t i = 0; i < p; ++i) {
            dm[i] = pm[i]; dv[i] = pv[i];
            dg[i] = server_step(opt, pg[i], pa[i], dm[i], dv[i], sp);
          }
          return py::make_tuple(go, mo, vo);
        },
        py::arg("g"), py::arg("a"), py::arg("m"), py::arg("v"), py::arg("opt"), py::arg("params"));
  // robust_combine over every coordinate: values float32 [K][P] (K in 1..64) -> float32 [P], trim
  // clamped to (K - 1) / 2 -- a trim of 64 or more is the coordinate-wise median
  m.def("aggregate_coordinates",
        [](const py::array_t<float, py::array::c_style | py::array::forcecast>& values, int trim) {
          if (values.ndim() != 2 || values.shape(0) < 1 || values.shape(0) > kCMaxRanks)
            throw std::invalid_argument("values must be float32 [K][P] with 1 <= K <= 64");
          if (trim < 0) throw std::invalid_argument("trim must be >= 0");
          const int k = static_cast<int>(values.shape(0));
          const py::ssize_t p = values.shape(1);
          const int t = agg_trim(AGG_TRIMMED_MEAN, trim, k);
          py::array_t<float> out(p);
          const float* src = values.data();
          float* dst = out.mutable_data();
          float v[kCMaxRanks];
          for (py::ssize_t i = 0; i < p; ++i) {
            for (int j = 0; j < k; ++j) v[j] = src[j * p + i];
            dst[i] = robust_combine<kCMaxRanks>(v, k, t);
          }
          return out;
        },
        py::arg("values"), py::arg("trim"));

  // Stand-alone access to the shared decision procedure (differential tests vs the oracle
  // and vs the device kernel).
  m.def("run_consensus", [](int n_ranks, int n_comm, int n_aggregate, bool weight_by_score,
                            std::vector<uint32_t> role, std::vector<int> admitted,
                            std::vector<std::vector<float>> score,
                            std::vector<std::vector<int>> scored, std::vector<uint32_t> n_samples,
                            std::vector<float> avg_cost) {
    ConsensusIn<kCMaxRanks> in;
    std::memset(&in, 0, sizeof(in));
    ConsensusOut<kCMaxRanks> out;
    std::memset(&out, 0, sizeof(out));
    in.n_ranks = n_ranks; in.n_comm = n_comm; in.n_aggregate = n_aggregate;
    in.weight_by_score = weight_by_score ? 1 : 0;
    for (int r = 0; r < n_ranks; ++r) {
      in.role[r] = role.at(r); in.admitted[r] = admitted.at(r) ? 1 : 0;
      in.n_samples[r] = n_samples.at(r); in.avg_cost[r] = avg_cost.at(r);
      for (int t = 0; t < n_ranks; ++t) {
        in.scored[r][t] = scored.at(r).at(t) ? 1 : 0;
        in.score[r][t] = score.at(r).at(t);
      }
    }
    run_consensus<kCMaxRanks>(in, out);
    py::dict d;
    std::vector<float> med(out.median, out.median + n_ranks), w(out.weight, out.weight + n_ranks);
    std::vector<int> order(out.order, out.order + out.n_ranked);
    std::vector<int> sel;
    for (int r = 0; r < n_ranks; ++r) if (out.selected[r]) sel.push_back(r);
    std::vector<uint32_t> ra(out.role_after, out.role_after + n_ranks);
    d["median"] = med; d["weight"] = w; d["order"] = order; d["selected"] = sel;
    d["role_after"] = ra; d["global_loss"] = out.global_loss;
    return d;
  });
}
