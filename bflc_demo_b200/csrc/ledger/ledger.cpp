// See ledger.hpp for the reference parity map.
#include "ledger.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <stdexcept>

#include "consensus_math.hpp"

namespace bflc {

// ------------------------------------------------------------------ sha256
namespace {
constexpr uint32_t kK[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4,
    0xab1c5ed5, 0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe,
    0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f,
    0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7,
    0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc,
    0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b,
    0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116,
    0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
    0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7,
    0xc67178f2};
inline uint32_t rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }

void sha_block(uint32_t h[8], const uint8_t* p) {
  uint32_t w[64];
  for (int i = 0; i < 16; ++i)
    w[i] = (uint32_t(p[4 * i]) << 24) | (uint32_t(p[4 * i + 1]) << 16) |
           (uint32_t(p[4 * i + 2]) << 8) | uint32_t(p[4 * i + 3]);
  for (int i = 16; i < 64; ++i) {
    const uint32_t s0 = rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3);
    const uint32_t s1 = rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
    w[i] = w[i - 16] + s0 + w[i - 7] + s1;
  }
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
  for (int i = 0; i < 64; ++i) {
    const uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25);
    const uint32_t ch = (e & f) ^ (~e & g);
    const uint32_t t1 = hh + S1 + ch + kK[i] + w[i];
    const uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22);
    const uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
    const uint32_t t2 = S0 + mj;
    hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

// little-endian binary writer / reader used for block hashing and snapshots
struct Writer {
  std::string buf;
  template <typename T>
  void pod(const T& v) { buf.append(reinterpret_cast<const char*>(&v), sizeof(T)); }
  template <typename T>
  void vec(const std::vector<T>& v) {
    pod<uint64_t>(v.size());
    if (!v.empty()) buf.append(reinterpret_cast<const char*>(v.data()), sizeof(T) * v.size());
  }
  void hash(const Hash256& h) { buf.append(reinterpret_cast<const char*>(h.data()), 32); }
};
struct Reader {
  const std::string& buf;
  size_t pos = 0;
  explicit Reader(const std::string& b) : buf(b) {}
  void need(size_t n) const {   // overflow-safe: pos <= buf.size() always holds
    if (n > buf.size() - pos) throw std::runtime_error("ledger snapshot truncated");
  }
  template <typename T>
  T pod() {
    need(sizeof(T));
    T v;
    std::memcpy(&v, buf.data() + pos, sizeof(T));
    pos += sizeof(T);
    return v;
  }
  template <typename T>
  std::vector<T> vec() {
    const uint64_t n = pod<uint64_t>();
    if (n > (buf.size() - pos) / sizeof(T)) throw std::runtime_error("ledger snapshot truncated");
    std::vector<T> v(n);
    if (n) std::memcpy(v.data(), buf.data() + pos, n * sizeof(T));
    pos += n * sizeof(T);
    return v;
  }
  Hash256 hash() {
    need(32);
    Hash256 h;
    std::memcpy(h.data(), buf.data() + pos, 32);
    pos += 32;
    return h;
  }
};

void write_block(Writer& w, const Block& b, bool with_hash) {
  w.pod(b.index); w.pod<int32_t>(b.epoch); w.hash(b.prev_hash);
  w.vec(b.role_before); w.vec(b.role_after); w.vec(b.admitted); w.vec(b.committee);
  w.pod<uint64_t>(b.scores.size());
  for (const auto& row : b.scores) w.vec(row);
  w.vec(b.median); w.vec(b.selected); w.vec(b.weight);
  w.pod(b.global_loss); w.hash(b.model_hash); w.pod(b.device_digest); w.pod(b.from_device);
  if (with_hash) w.hash(b.hash);
}
Block read_block(Reader& r) {
  Block b;
  b.index = r.pod<uint64_t>(); b.epoch = r.pod<int32_t>(); b.prev_hash = r.hash();
  b.role_before = r.vec<uint32_t>(); b.role_after = r.vec<uint32_t>();
  b.admitted = r.vec<int>(); b.committee = r.vec<int>();
  const uint64_t nrows = r.pod<uint64_t>();
  for (uint64_t i = 0; i < nrows; ++i) b.scores.push_back(r.vec<float>());
  b.median = r.vec<float>(); b.selected = r.vec<int>(); b.weight = r.vec<float>();
  b.global_loss = r.pod<float>(); b.model_hash = r.hash();
  b.device_digest = r.pod<uint64_t>(); b.from_device = r.pod<uint8_t>();
  b.hash = r.hash();
  return b;
}

uint64_t splitmix64(uint64_t& s) {
  uint64_t z = (s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

using CIn = ConsensusIn<kCMaxRanks>;
using COut = ConsensusOut<kCMaxRanks>;
}  // namespace

Hash256 sha256(const void* data, size_t n) {
  uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a,
                   0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
  const uint8_t* p = static_cast<const uint8_t*>(data);
  size_t full = n / 64;
  for (size_t i = 0; i < full; ++i) sha_block(h, p + 64 * i);
  uint8_t tail[128] = {0};
  const size_t rem = n - full * 64;
  std::memcpy(tail, p + full * 64, rem);
  tail[rem] = 0x80;
  const size_t tl = rem + 9 <= 64 ? 64 : 128;
  const uint64_t bits = static_cast<uint64_t>(n) * 8;
  for (int i = 0; i < 8; ++i) tail[tl - 1 - i] = static_cast<uint8_t>(bits >> (8 * i));
  sha_block(h, tail);
  if (tl == 128) sha_block(h, tail + 64);
  Hash256 out;
  for (int i = 0; i < 8; ++i) {
    out[4 * i] = h[i] >> 24; out[4 * i + 1] = h[i] >> 16; out[4 * i + 2] = h[i] >> 8;
    out[4 * i + 3] = h[i];
  }
  return out;
}

std::string hex(const Hash256& h) {
  static const char* d = "0123456789abcdef";
  std::string s(64, '0');
  for (int i = 0; i < 32; ++i) { s[2 * i] = d[h[i] >> 4]; s[2 * i + 1] = d[h[i] & 15]; }
  return s;
}

const char* status_name(Status s) {
  switch (s) {
    case Status::OK: return "OK";
    case Status::NOT_STARTED: return "NOT_STARTED";
    case Status::STALE_EPOCH: return "STALE_EPOCH";
    case Status::DUPLICATE: return "DUPLICATE";
    case Status::QUOTA_FULL: return "QUOTA_FULL";
    case Status::NOT_COMMITTEE: return "NOT_COMMITTEE";
    case Status::UNKNOWN_CLIENT: return "UNKNOWN_CLIENT";
    case Status::BAD_PAYLOAD: return "BAD_PAYLOAD";
    case Status::AGGREGATED: return "AGGREGATED";
    case Status::NOT_TRAINER: return "NOT_TRAINER";
    case Status::NOT_READY: return "NOT_READY";
  }
  return "?";
}

int LedgerConfig::dp_mode() const { return dp_mode_of(dp_clip, dp_noise); }
int LedgerConfig::dp_kernel_mode() const { return bflc::dp_kernel_mode(dp_mode(), dp_adaptive()); }

void dp_gauss_fill(uint64_t seed, uint32_t epoch, uint64_t first, float* out, size_t n) {
  float z[4];
  uint64_t have = ~0ull;   // float4 index whose four normals z holds
  for (size_t k = 0; k < n; ++k) {
    const uint64_t i = first + k;
    if (i / 4 != have) {
      have = i / 4;
      dp_gauss4(seed, epoch, have, z, kDpSite);
    }
    out[k] = z[i % 4];
  }
}

std::string LedgerConfig::validate() const {
  if (client_num < 1 || client_num > kCMaxRanks) return "client_num must be in [1, 64]";
  if (comm_count < 1) return "comm_count must be >= 1";
  if (aggregate_count < 1) return "aggregate_count must be >= 1";
  if (aggregate_count > needed_update_count) return "aggregate_count > needed_update_count";
  if (model_size < 1) return "model_size must be >= 1";
  if (!(learning_rate > 0.f)) return "learning_rate must be > 0";
  if (aggregation != AGG_FEDAVG && aggregation != AGG_MEDIAN && aggregation != AGG_TRIMMED_MEAN)
    return "aggregation must be 0 (FedAvg), 1 (median) or 2 (trimmed mean)";
  if (aggregation == AGG_TRIMMED_MEAN && (trim < 1 || 2 * trim >= aggregate_count))
    return "trimmed mean needs 1 <= trim and 2 * trim < aggregate_count";
  if (aggregation != AGG_FEDAVG && weight_by_score) return "weight_by_score needs the FedAvg rule";
  if (const char* e = server_opt_check(server_opt, server_lr, server_beta1, server_beta2, server_tau); *e) return e;
  if (dp_clip == 0.f && dp_noise != 0.f) return "dp_noise needs dp_clip > 0";
  if (const char* e = dp_check(dp_mode(), dp_clip, dp_noise, aggregation); *e) return e;
  if (const char* e = dp_adapt_check(dp_mode(), dp_noise, dp_clip_quantile, dp_clip_lr, dp_count_noise); *e) return e;
  if (solo) {
    if (comm_count > client_num) return "comm_count > client_num";
    if (needed_update_count > client_num) return "needed_update_count > client_num";
    return "";
  }
  // comm_count > needed_update_count is allowed (BASELINE config #4: committee 5 of 8): the
  // election takes every scored trainer and refills from the outgoing committee.
  if (needed_update_count > client_num - comm_count)
    return "needed_update_count > client_num - comm_count (not enough trainers)";
  return "";
}

Ledger::Ledger(const LedgerConfig& cfg) : cfg_(cfg) {
  const std::string err = cfg.validate();
  if (!err.empty()) throw std::invalid_argument("LedgerConfig: " + err);
  global_.assign(static_cast<size_t>(cfg.model_size), 0.f);  // InitGlobalModel, C:321-346
  clip_now_ = cfg.dp_clip;
}

void Ledger::log(std::string s) {
  if (log_.size() < 4096) log_.push_back(std::move(s));
}

const MethodInfo* method_table(int* n) {
  static const MethodInfo kTable[] = {
      {Method::RegisterNode, "RegisterNode()", false},
      {Method::QueryState, "QueryState()", true},
      {Method::QueryGlobalModel, "QueryGlobalModel()", true},
      {Method::UploadLocalUpdate, "UploadLocalUpdate(string,int256)", false},
      {Method::UploadScores, "UploadScores(int256,string)", false},
      {Method::QueryAllUpdates, "QueryAllUpdates()", true},
  };
  if (n) *n = 6;
  return kTable;
}

Method method_from_signature(const std::string& s) {
  int n = 0;
  const MethodInfo* t = method_table(&n);
  for (int i = 0; i < n; ++i) {
    const std::string sig = t[i].signature;
    if (s == sig || s == sig.substr(0, sig.find('('))) return t[i].id;
  }
  return Method::Unknown;
}

Status Ledger::RegisterNode(int client) {
  std::lock_guard<std::mutex> g(mu_);
  ++ctr_.calls;
  if (client < 0 || client >= cfg_.client_num) return Status::UNKNOWN_CLIENT;
  if (role_.count(client)) return Status::OK;  // idempotent, C:171
  role_[client] = ROLE_TRAINER;
  registered_.push_back(client);
  ++ctr_.register_ok;
  if (static_cast<int>(role_.size()) == cfg_.client_num && epoch_ == kEpochNotStarted) {
    // C:175-186: once everybody registered pick the first committee and start epoch 0.
    std::vector<int> ids;
    for (auto& kv : role_) ids.push_back(kv.first);
    if (cfg_.seed != 0) {
      uint64_t s = cfg_.seed;
      for (size_t i = ids.size(); i > 1; --i) std::swap(ids[i - 1], ids[splitmix64(s) % i]);
    }
    if (cfg_.solo) {
      for (auto& kv : role_) kv.second = ROLE_TRAINER | ROLE_COMM;
    } else {
      for (int i = 0; i < cfg_.comm_count; ++i) role_[ids[static_cast<size_t>(i)]] = ROLE_COMM;
    }
    epoch_ = 0;
    log("all " + std::to_string(cfg_.client_num) + " nodes registered, epoch 0 starts");
  }
  return Status::OK;
}

std::pair<uint32_t, int> Ledger::QueryState(int client) {
  std::lock_guard<std::mutex> g(mu_);
  ++ctr_.calls; ++ctr_.queries;
  auto it = role_.find(client);
  return {it == role_.end() ? static_cast<uint32_t>(ROLE_TRAINER) : it->second, epoch_};
}

std::pair<std::vector<float>, int> Ledger::QueryGlobalModel() {
  std::lock_guard<std::mutex> g(mu_);
  ++ctr_.calls; ++ctr_.queries;
  return {global_, epoch_};
}

Status Ledger::UploadLocalUpdate(int client, const std::vector<float>& delta, UpdateMeta meta,
                                 int ep) {
  std::lock_guard<std::mutex> g(mu_);
  ++ctr_.calls;
  auto reject = [&](Status s) {
    ++ctr_.uploads_rejected;
    log("the update of local model is not collected (" + std::string(status_name(s)) + ")");
    return s;
  };
  if (epoch_ == kEpochNotStarted) return reject(Status::NOT_STARTED);
  if (ep != epoch_) return reject(Status::STALE_EPOCH);
  auto it = role_.find(client);
  if (it == role_.end()) return reject(Status::UNKNOWN_CLIENT);
  if (!(it->second & ROLE_TRAINER)) return reject(Status::NOT_TRAINER);
  if (updates_.count(client)) return reject(Status::DUPLICATE);
  if (static_cast<int>(updates_.size()) >= cfg_.needed_update_count)
    return reject(Status::QUOTA_FULL);
  if (static_cast<int64_t>(delta.size()) != cfg_.model_size) return reject(Status::BAD_PAYLOAD);
  LocalUpdate u;
  u.sender = client; u.delta = delta; u.meta = meta; u.arrival = arrivals_++;
  updates_.emplace(client, std::move(u));
  ++ctr_.uploads_ok;
  log("the update of local model is collected");
  return Status::OK;
}

std::vector<LocalUpdate> Ledger::QueryAllUpdates() {
  std::lock_guard<std::mutex> g(mu_);
  ++ctr_.calls; ++ctr_.queries;
  std::vector<LocalUpdate> out;
  if (static_cast<int>(updates_.size()) < cfg_.needed_update_count) return out;  // C:304-307
  for (auto& kv : updates_) out.push_back(kv.second);
  std::sort(out.begin(), out.end(),
            [](const LocalUpdate& a, const LocalUpdate& b) { return a.arrival < b.arrival; });
  return out;
}

Status Ledger::UploadScores(int client, int ep, const std::map<int, float>& scores) {
  std::lock_guard<std::mutex> g(mu_);
  ++ctr_.calls;
  auto reject = [&](Status s) { ++ctr_.scores_rejected; return s; };
  if (epoch_ == kEpochNotStarted) return reject(Status::NOT_STARTED);
  if (ep != epoch_) return reject(Status::STALE_EPOCH);
  auto it = role_.find(client);
  if (it == role_.end() || !(it->second & ROLE_COMM)) return reject(Status::NOT_COMMITTEE);
  if (static_cast<int>(updates_.size()) < cfg_.needed_update_count)
    return reject(Status::NOT_READY);
  std::map<int, float> row;
  for (auto& kv : scores) {
    if (!updates_.count(kv.first)) continue;  // only admitted trainers can be scored
    if (!std::isfinite(kv.second)) return reject(Status::BAD_PAYLOAD);
    row[kv.first] = kv.second;
  }
  // A repeated upload replaces the row and is NOT counted twice (the reference increments
  // score_count on duplicates, C:279-289 -- a latent bug that is deliberately not emulated).
  scores_[client] = std::move(row);
  ++ctr_.scores_ok;
  log(std::to_string(scores_.size()) + " scores has been uploaded");
  if (static_cast<int>(scores_.size()) == cfg_.comm_count) {
    aggregate_locked();
    return Status::AGGREGATED;
  }
  return Status::OK;
}

void Ledger::aggregate_locked() {
  // Aggregate, C:349-456
  CIn in;
  std::memset(&in, 0, sizeof(in));
  COut out;
  std::memset(&out, 0, sizeof(out));
  const int n = cfg_.client_num;
  in.n_ranks = n;
  in.n_comm = cfg_.comm_count;
  in.n_aggregate = cfg_.aggregate_count;
  in.weight_by_score = cfg_.weight_by_score;
  for (auto& kv : role_) in.role[kv.first] = kv.second;
  for (auto& kv : updates_) {
    in.admitted[kv.first] = 1;
    in.n_samples[kv.first] = kv.second.meta.n_samples;
    in.avg_cost[kv.first] = kv.second.meta.avg_cost;
  }
  for (auto& row : scores_)
    for (auto& kv : row.second) {
      in.scored[row.first][kv.first] = 1;
      in.score[row.first][kv.first] = kv.second;
    }
  run_consensus<kCMaxRanks>(in, out);

  // DP (consensus_math.hpp): update t's model change is lr * delta_t; its norm is that of the fp32
  // products, the squares summed in fp64 in ascending index order, and a clipped update enters the
  // rule as s_t * delta_t
  const int dp = cfg_.dp_mode();
  const bool adaptive = cfg_.dp_adaptive();
  const float clip = adaptive ? clip_now_ : cfg_.dp_clip;   // C_t
  uint32_t unclipped = 0;                                  // adaptive: b, the count dp_scale leaves alone
  std::vector<const float*> dsrc(static_cast<size_t>(n), nullptr);
  std::vector<std::vector<float>> clipped;
  clipped.reserve(static_cast<size_t>(n));
  for (int t = 0; t < n; ++t) {
    if (!out.selected[t]) continue;
    const std::vector<float>& d = updates_.at(t).delta;
    dsrc[static_cast<size_t>(t)] = d.data();
    if (dp == DP_OFF) continue;
    double sum = 0.0;
    for (float x : d) {
      const double c = so_mul(cfg_.learning_rate, x);
      sum += c * c;
    }
    const float nrm = dp_norm(sum);
    const float s = dp_scale(nrm, clip);
    unclipped += dp_bits(nrm) <= dp_bits(clip) ? 1u : 0u;
    if (dp_bits(s) == 0x3F800000u) continue;
    clipped.emplace_back(d.size());
    for (size_t i = 0; i < d.size(); ++i) clipped.back()[i] = so_mul(s, d[i]);
    dsrc[static_cast<size_t>(t)] = clipped.back().data();
  }

  // steps 2-4: global -= lr * sum_k w_k * delta_k, fixed (ascending id) order; a robust rule
  // puts the coordinate-wise trimmed mean / median of the selected deltas in place of the sum
  std::vector<float> total(global_.size(), 0.f);
  if (cfg_.aggregation == AGG_FEDAVG) {
    for (int t = 0; t < n; ++t) {
      if (!out.selected[t]) continue;
      const float w = out.weight[t];
      const float* d = dsrc[static_cast<size_t>(t)];
      for (size_t i = 0; i < total.size(); ++i) total[i] = std::fmaf(w, d[i], total[i]);
    }
  } else if (out.n_selected > 0) {
    std::vector<const float*> sel;
    for (int t = 0; t < n; ++t)
      if (out.selected[t]) sel.push_back(dsrc[static_cast<size_t>(t)]);
    const int k = static_cast<int>(sel.size());
    const int trim = agg_trim(cfg_.aggregation, cfg_.trim, k);
    float v[kCMaxRanks];
    for (size_t i = 0; i < total.size(); ++i) {
      for (int j = 0; j < k; ++j) v[j] = sel[static_cast<size_t>(j)][i];
      total[i] = robust_combine<kCMaxRanks>(v, k, trim);
    }
  }
  // DP noise on the aggregate (FedAvg, something selected): a_i + sigma * xi_i, sigma = (z * C) * max w
  std::vector<float> noise;
  float sigma = 0.f;
  if (dp == DP_NOISE && out.n_selected > 0) {
    uint32_t wmax = 0;
    for (int t = 0; t < n; ++t)
      if (out.selected[t] && dp_bits(out.weight[t]) > wmax) wmax = dp_bits(out.weight[t]);
    const float zmul = adaptive ? dp_noise_split(cfg_.dp_noise, cfg_.dp_count_noise) : cfg_.dp_noise;
    sigma = so_mul(so_mul(zmul, clip), dp_float(wmax));
    noise.resize(global_.size());
    dp_gauss_fill(cfg_.dp_seed, static_cast<uint32_t>(epoch_), 0, noise.data(), noise.size());
  }
  if (cfg_.server_opt == SOPT_NONE) {
    for (size_t i = 0; i < global_.size(); ++i) global_[i] -= cfg_.learning_rate * total[i];
    for (size_t i = 0; i < noise.size(); ++i) global_[i] = so_add(global_[i], so_mul(sigma, noise[i]));
  } else {
    // the aggregate a is exactly the new model the line above gives; the server step moves from the
    // current model along d = global - a (nothing selected: model and state stay as they are)
    if (server_m_.empty()) {
      server_m_.assign(global_.size(), 0.f);
      if (server_state_vectors(cfg_.server_opt) == 2) server_v_.assign(global_.size(), 0.f);
    }
    if (out.n_selected > 0) {
      const ServerOptParams p = server_opt_params(cfg_.server_lr, cfg_.server_beta1, cfg_.server_beta2, cfg_.server_tau);
      float v_unused = 0.f;
      for (size_t i = 0; i < global_.size(); ++i) {
        float a = global_[i] - cfg_.learning_rate * total[i];
        if (!noise.empty()) a = so_add(a, so_mul(sigma, noise[i]));
        float& v = server_v_.empty() ? v_unused : server_v_[i];
        global_[i] = server_step(cfg_.server_opt, global_[i], a, server_m_[i], v, p);
      }
    }
  }

  // adaptive clipping: C_{t+1} from this round's noised count, after the combine used C_t
  if (adaptive) {
    last_clip_.clip = clip;
    last_clip_.n_sel = out.n_selected;
    last_clip_.count = dp_noised_count(unclipped, out.n_selected, dp == DP_NOISE ? cfg_.dp_count_noise : 0.f,
                                       cfg_.dp_seed, static_cast<uint32_t>(epoch_));
    if (out.n_selected > 0)
      clip_now_ = dp_clip_next(clip, last_clip_.count, out.n_selected, cfg_.dp_clip_quantile, cfg_.dp_clip_lr);
  }

  Block b;
  b.epoch = epoch_;
  b.role_before.assign(static_cast<size_t>(n), 0);
  b.role_after.assign(static_cast<size_t>(n), 0);
  for (int r = 0; r < n; ++r) {
    b.role_before[static_cast<size_t>(r)] = in.role[r];
    b.role_after[static_cast<size_t>(r)] = out.role_after[r];
  }
  std::vector<const LocalUpdate*> adm;
  for (auto& kv : updates_) adm.push_back(&kv.second);
  std::sort(adm.begin(), adm.end(),
            [](const LocalUpdate* a, const LocalUpdate* c) { return a->arrival < c->arrival; });
  for (auto* u : adm) { b.admitted.push_back(u->sender); b.median.push_back(out.median[u->sender]); }
  for (auto& row : scores_) {
    b.committee.push_back(row.first);
    std::vector<float> r;
    for (int t : b.admitted) {
      auto f = row.second.find(t);
      r.push_back(f == row.second.end() ? std::nanf("") : f->second);
    }
    b.scores.push_back(std::move(r));
  }
  for (int t = 0; t < n; ++t)
    if (out.selected[t]) { b.selected.push_back(t); b.weight.push_back(out.weight[t]); }
  b.global_loss = out.global_loss;
  b.model_hash = sha256(global_.data(), global_.size() * sizeof(float));
  last_loss_ = out.global_loss;
  log("the " + std::to_string(epoch_) + " epoch , global loss : " + std::to_string(out.global_loss));

  for (int r = 0; r < n; ++r)
    if (role_.count(r)) role_[r] = out.role_after[r];
  updates_.clear();
  scores_.clear();
  epoch_ += 1;
  ++ctr_.aggregations;
  append_block_locked(std::move(b));
}

Hash256 Ledger::hash_block(const Block& b) const {
  Writer w;
  write_block(w, b, /*with_hash=*/false);
  return sha256(w.buf.data(), w.buf.size());
}

void Ledger::append_block_locked(Block&& b) {
  b.index = chain_.size();
  if (!chain_.empty()) b.prev_hash = chain_.back().hash;
  b.hash = hash_block(b);
  chain_.push_back(std::move(b));
}

void Ledger::Bootstrap(const std::vector<uint32_t>& roles) {
  std::lock_guard<std::mutex> g(mu_);
  if (static_cast<int>(roles.size()) != cfg_.client_num)
    throw std::invalid_argument("Bootstrap: one role per client required");
  role_.clear(); registered_.clear();
  for (int r = 0; r < cfg_.client_num; ++r) {
    role_[r] = roles[static_cast<size_t>(r)];
    registered_.push_back(r);
  }
  epoch_ = 0;
}

std::string Ledger::AppendDeviceRound(const DeviceRound& r) {
  std::lock_guard<std::mutex> g(mu_);
  const int n = cfg_.client_num;
  if (r.epoch != epoch_)
    return "epoch mismatch: device " + std::to_string(r.epoch) + " host " + std::to_string(epoch_);
  // the device path keeps its masks in 32-bit words (kMaxRanks = 8 today)
  if (n > 32) return "device rounds support at most 32 clients";
  const size_t un = static_cast<size_t>(n);
  if (r.role_before.size() < un || r.role_after.size() < un || r.score_rows.size() < un ||
      r.scored_mask.size() < un || r.n_samples.size() < un || r.avg_cost.size() < un)
    return "short device record";
  for (size_t c = 0; c < un; ++c)
    if (r.score_rows[c].size() < un) return "short score row in device record";
  CIn in;
  std::memset(&in, 0, sizeof(in));
  COut out;
  std::memset(&out, 0, sizeof(out));
  in.n_ranks = n; in.n_comm = cfg_.comm_count; in.n_aggregate = cfg_.aggregate_count;
  in.weight_by_score = r.weight_by_score;
  for (int c = 0; c < n; ++c) {
    if (role_.at(c) != r.role_before[static_cast<size_t>(c)])
      return "role_before mismatch at rank " + std::to_string(c);
    in.role[c] = r.role_before[static_cast<size_t>(c)];
    in.admitted[c] = (r.admitted_mask >> c) & 1u;
    in.n_samples[c] = r.n_samples[static_cast<size_t>(c)];
    in.avg_cost[c] = r.avg_cost[static_cast<size_t>(c)];
    for (int t = 0; t < n; ++t) {
      in.scored[c][t] = (r.scored_mask[static_cast<size_t>(c)] >> t) & 1u;
      in.score[c][t] = r.score_rows[static_cast<size_t>(c)][static_cast<size_t>(t)];
    }
  }
  run_consensus<kCMaxRanks>(in, out);  // re-execute the election on the host
  uint32_t sel = 0;
  for (int t = 0; t < n; ++t)
    if (out.selected[t]) sel |= 1u << t;
  if (sel != r.selected_mask) return "selected set mismatch";
  for (int c = 0; c < n; ++c)
    if (out.role_after[c] != r.role_after[static_cast<size_t>(c)])
      return "re-election mismatch at rank " + std::to_string(c);
  if (std::fabs(out.global_loss - r.global_loss) > 1e-5f * (1.f + std::fabs(out.global_loss)))
    return "global_loss mismatch";
  const uint32_t word = agg_word(cfg_.aggregation, cfg_.trim, cfg_.server_opt, cfg_.dp_kernel_mode());
  if ((r.agg & 0xFFFFu) != (word & 0xFFFFu))
    return "aggregation rule mismatch: device word " + std::to_string(r.agg) + " config " + std::to_string(word);
  if ((r.agg & 0xFFFFFFu) != (word & 0xFFFFFFu))
    return "server optimizer mismatch: device word " + std::to_string(r.agg) + " config " + std::to_string(word);
  if (r.agg != word)
    return "differential privacy mismatch: device word " + std::to_string(r.agg) + " config " + std::to_string(word);
  // adaptive clipping: the record's C_t must be the host's, its noised count one that b in [0, n_sel]
  // (with this epoch's count noise) gives; then the host takes the same step to C_{t+1}
  float next_clip = clip_now_;
  if (cfg_.dp_adaptive()) {
    const std::string at = " at epoch " + std::to_string(r.epoch);
    int n_sel = 0;
    for (int t = 0; t < n; ++t) n_sel += out.selected[t] ? 1 : 0;
    if (!r.has_clip) return "clip trajectory mismatch: no clip record" + at;
    if (dp_bits(r.clip) != dp_bits(clip_now_))
      return "clip trajectory mismatch: device clip " + std::to_string(r.clip) + " host " + std::to_string(clip_now_) + at;
    if (r.n_sel != static_cast<uint32_t>(n_sel)) return "clip trajectory mismatch: selected count" + at;
    const float sb = cfg_.dp_mode() == DP_NOISE ? cfg_.dp_count_noise : 0.f;
    bool ok = false;
    for (int b = 0; b <= n_sel && !ok; ++b)
      ok = dp_bits(dp_noised_count(static_cast<uint32_t>(b), n_sel, sb, cfg_.dp_seed, static_cast<uint32_t>(r.epoch))) ==
           dp_bits(r.count);
    if (!ok) return "clip trajectory mismatch: noised count " + std::to_string(r.count) + " is no count of the selected updates" + at;
    if (n_sel > 0) next_clip = dp_clip_next(clip_now_, r.count, n_sel, cfg_.dp_clip_quantile, cfg_.dp_clip_lr);
    last_clip_.clip = clip_now_;
    last_clip_.count = r.count;
    last_clip_.n_sel = n_sel;
  }

  Block b;
  b.epoch = epoch_;
  b.from_device = 1;
  b.device_digest = r.model_digest;
  b.role_before.assign(r.role_before.begin(), r.role_before.begin() + n);
  b.role_after.assign(r.role_after.begin(), r.role_after.begin() + n);
  for (int t = 0; t < n; ++t)
    if (in.admitted[t]) { b.admitted.push_back(t); b.median.push_back(out.median[t]); }
  for (int c = 0; c < n; ++c) {
    if (!(in.role[c] & ROLE_COMM)) continue;
    b.committee.push_back(c);
    std::vector<float> row;
    for (int t : b.admitted) row.push_back(in.scored[c][t] ? in.score[c][t] : std::nanf(""));
    b.scores.push_back(std::move(row));
  }
  for (int t = 0; t < n; ++t)
    if (out.selected[t]) { b.selected.push_back(t); b.weight.push_back(out.weight[t]); }
  b.global_loss = out.global_loss;
  last_loss_ = out.global_loss;
  for (int c = 0; c < n; ++c) role_[c] = out.role_after[c];
  clip_now_ = next_clip;
  epoch_ += 1;
  ++ctr_.aggregations;
  log("the " + std::to_string(b.epoch) + " epoch , global loss : " + std::to_string(b.global_loss));
  append_block_locked(std::move(b));
  return "";
}

int Ledger::epoch() const { std::lock_guard<std::mutex> g(mu_); return epoch_; }
float Ledger::dp_clip_now() const { std::lock_guard<std::mutex> g(mu_); return clip_now_; }
Ledger::ClipStep Ledger::last_clip_step() const { std::lock_guard<std::mutex> g(mu_); return last_clip_; }
std::pair<std::vector<float>, std::vector<float>> Ledger::server_state() const {
  std::lock_guard<std::mutex> g(mu_);
  return {server_m_, server_v_};
}
int Ledger::update_count() const { std::lock_guard<std::mutex> g(mu_); return (int)updates_.size(); }
int Ledger::score_count() const { std::lock_guard<std::mutex> g(mu_); return (int)scores_.size(); }
size_t Ledger::n_blocks() const { std::lock_guard<std::mutex> g(mu_); return chain_.size(); }
float Ledger::last_global_loss() const { std::lock_guard<std::mutex> g(mu_); return last_loss_; }
OpCounters Ledger::counters() const { std::lock_guard<std::mutex> g(mu_); return ctr_; }
std::vector<Block> Ledger::blocks() const { std::lock_guard<std::mutex> g(mu_); return chain_; }
std::vector<std::string> Ledger::drain_log() {
  std::lock_guard<std::mutex> g(mu_);
  std::vector<std::string> out;
  out.swap(log_);
  return out;
}
std::vector<uint32_t> Ledger::roles() const {
  std::lock_guard<std::mutex> g(mu_);
  std::vector<uint32_t> out(static_cast<size_t>(cfg_.client_num), 0);
  for (auto& kv : role_) out[static_cast<size_t>(kv.first)] = kv.second;
  return out;
}

Hash256 Ledger::state_hash() const {
  std::lock_guard<std::mutex> g(mu_);
  Writer w;
  w.pod<int32_t>(epoch_);
  for (auto& kv : role_) { w.pod<int32_t>(kv.first); w.pod(kv.second); }
  w.vec(global_);
  if (cfg_.server_opt != SOPT_NONE) { w.vec(server_m_); w.vec(server_v_); }
  if (cfg_.dp_mode() != DP_OFF) {   // not the seed (see snapshot())
    w.pod<uint32_t>(static_cast<uint32_t>(cfg_.dp_mode())); w.pod(cfg_.dp_clip); w.pod(cfg_.dp_noise);
  }
  if (cfg_.dp_adaptive()) {
    w.pod(cfg_.dp_clip_quantile); w.pod(cfg_.dp_clip_lr); w.pod(cfg_.dp_count_noise); w.pod(clip_now_);
  }
  for (auto& kv : updates_) { w.pod<int32_t>(kv.first); w.vec(kv.second.delta); }
  for (auto& row : scores_)
    for (auto& kv : row.second) { w.pod<int32_t>(row.first); w.pod<int32_t>(kv.first); w.pod(kv.second); }
  if (!chain_.empty()) w.hash(chain_.back().hash);
  return sha256(w.buf.data(), w.buf.size());
}

bool Ledger::verify_chain() const {
  std::lock_guard<std::mutex> g(mu_);
  Hash256 prev{};
  for (size_t i = 0; i < chain_.size(); ++i) {
    const Block& b = chain_[i];
    if (b.index != i || b.prev_hash != prev || hash_block(b) != b.hash) return false;
    prev = b.hash;
  }
  return true;
}

std::string Ledger::snapshot() const {
  std::lock_guard<std::mutex> g(mu_);
  Writer w;
  w.pod<uint32_t>(0xB1F1C0DEu);  // magic
  // version 1: FedAvg (the original format, byte for byte); version 2 adds the aggregation rule;
  // version 3 (any server optimizer) adds the rule word, the optimizer word and its four
  // hyperparameters, and the state vectors after the global model (empty before the first host
  // aggregation); version 4 (DP on) has version 3's fields for any optimizer, none included, then the
  // DP mode word and the fp32 clip and noise multiplier.  The DP seed is deliberately not written: the
  // snapshot is the replicated ledger state, and whoever holds the seed can regenerate the noise and
  // subtract it.  It is kept with the engine checkpoint instead, and restore() takes it back.  Version 5
  // (adaptive clipping) is version 4 followed by the fp32 quantile, clip rate, count noise and current clip.
  const bool robust = cfg_.aggregation != AGG_FEDAVG;
  const bool opt = cfg_.server_opt != SOPT_NONE;
  const bool dp = cfg_.dp_mode() != DP_OFF;
  const bool adaptive = cfg_.dp_adaptive();
  w.pod<uint32_t>(adaptive ? 5 : dp ? 4 : opt ? 3 : robust ? 2 : 1);
  w.pod<int32_t>(cfg_.client_num); w.pod<int32_t>(cfg_.comm_count);
  w.pod<int32_t>(cfg_.aggregate_count); w.pod<int32_t>(cfg_.needed_update_count);
  w.pod(cfg_.learning_rate); w.pod<int64_t>(cfg_.model_size);
  w.pod<int32_t>(cfg_.weight_by_score); w.pod<int32_t>(cfg_.solo); w.pod<uint64_t>(cfg_.seed);
  if (robust || opt || dp) w.pod<uint32_t>(agg_word(cfg_.aggregation, cfg_.trim));
  if (opt || dp) {
    w.pod<uint32_t>(static_cast<uint32_t>(cfg_.server_opt));
    w.pod(cfg_.server_lr); w.pod(cfg_.server_beta1); w.pod(cfg_.server_beta2); w.pod(cfg_.server_tau);
  }
  if (dp) {
    w.pod<uint32_t>(static_cast<uint32_t>(cfg_.dp_mode()));
    w.pod(cfg_.dp_clip); w.pod(cfg_.dp_noise);
  }
  if (adaptive) {
    w.pod(cfg_.dp_clip_quantile); w.pod(cfg_.dp_clip_lr); w.pod(cfg_.dp_count_noise); w.pod(clip_now_);
  }
  w.pod<int32_t>(epoch_);
  w.vec(global_);
  if (opt) { w.vec(server_m_); w.vec(server_v_); }
  w.vec(registered_);
  w.pod<uint64_t>(role_.size());
  for (auto& kv : role_) { w.pod<int32_t>(kv.first); w.pod(kv.second); }
  w.pod<uint64_t>(updates_.size());
  for (auto& kv : updates_) {
    w.pod<int32_t>(kv.first); w.vec(kv.second.delta); w.pod(kv.second.meta.n_samples);
    w.pod(kv.second.meta.avg_cost); w.pod(kv.second.arrival);
  }
  w.pod<uint64_t>(scores_.size());
  for (auto& row : scores_) {
    w.pod<int32_t>(row.first); w.pod<uint64_t>(row.second.size());
    for (auto& kv : row.second) { w.pod<int32_t>(kv.first); w.pod(kv.second); }
  }
  w.pod(arrivals_); w.pod(last_loss_);
  w.pod<uint64_t>(chain_.size());
  for (auto& b : chain_) write_block(w, b, true);
  return w.buf;
}

std::unique_ptr<Ledger> Ledger::restore(const std::string& blob, uint64_t dp_seed) {
  Reader r(blob);
  if (r.pod<uint32_t>() != 0xB1F1C0DEu) throw std::runtime_error("not a ledger snapshot");
  const uint32_t version = r.pod<uint32_t>();
  if (version < 1 || version > 5) throw std::runtime_error("unsupported snapshot version");
  LedgerConfig c;
  c.client_num = r.pod<int32_t>(); c.comm_count = r.pod<int32_t>();
  c.aggregate_count = r.pod<int32_t>(); c.needed_update_count = r.pod<int32_t>();
  c.learning_rate = r.pod<float>(); c.model_size = r.pod<int64_t>();
  c.weight_by_score = r.pod<int32_t>(); c.solo = r.pod<int32_t>(); c.seed = r.pod<uint64_t>();
  if (version >= 2) {  // agg_word of the rule: version 2 a robust one, version 3 any
    const uint32_t word = r.pod<uint32_t>();
    c.aggregation = static_cast<int>(word & 0xFFu);
    c.trim = static_cast<int>(word >> 8);
    if ((version == 2 && c.aggregation == AGG_FEDAVG) || !agg_rule_valid(c.aggregation, c.trim) ||
        agg_word(c.aggregation, c.trim) != word)
      throw std::runtime_error("ledger snapshot: unknown aggregation rule or trim out of range");
  }
  if (version >= 3) {   // version 4: any optimizer, none included
    const uint32_t opt = r.pod<uint32_t>();
    if (opt < (version == 3 ? SOPT_MOMENTUM : SOPT_NONE) || opt > SOPT_YOGI)
      throw std::runtime_error("ledger snapshot: unknown server optimizer");
    c.server_opt = static_cast<int>(opt);
    c.server_lr = r.pod<float>(); c.server_beta1 = r.pod<float>();
    c.server_beta2 = r.pod<float>(); c.server_tau = r.pod<float>();
    if (*server_opt_check(c.server_opt, c.server_lr, c.server_beta1, c.server_beta2, c.server_tau))
      throw std::runtime_error("ledger snapshot: invalid server optimizer hyperparameters");
  }
  if (version >= 4) {
    const uint32_t mode = r.pod<uint32_t>();
    c.dp_clip = r.pod<float>(); c.dp_noise = r.pod<float>();
    c.dp_seed = dp_seed;
    if ((mode != DP_CLIP && mode != DP_NOISE) || c.dp_mode() != static_cast<int>(mode) ||
        *dp_check(c.dp_mode(), c.dp_clip, c.dp_noise, c.aggregation))
      throw std::runtime_error("ledger snapshot: invalid differential privacy fields");
  }
  float clip_now = c.dp_clip;
  if (version == 5) {
    c.dp_clip_quantile = r.pod<float>(); c.dp_clip_lr = r.pod<float>(); c.dp_count_noise = r.pod<float>();
    clip_now = r.pod<float>();
    if (!c.dp_adaptive() || *dp_adapt_check(c.dp_mode(), c.dp_noise, c.dp_clip_quantile, c.dp_clip_lr, c.dp_count_noise) ||
        !(clip_now >= kDpClipMin && clip_now <= kDpClipMax))
      throw std::runtime_error("ledger snapshot: invalid adaptive clipping fields");
  }
  auto LP = std::make_unique<Ledger>(c);
  Ledger& L = *LP;
  L.clip_now_ = clip_now;
  L.epoch_ = r.pod<int32_t>();
  L.global_ = r.vec<float>();
  if (c.server_opt != SOPT_NONE) {
    L.server_m_ = r.vec<float>(); L.server_v_ = r.vec<float>();
    // both empty (no host aggregation yet), or one model-sized vector per state vector
    const size_t p = static_cast<size_t>(c.model_size);
    const size_t want_v = server_state_vectors(c.server_opt) == 2 ? p : 0;
    if (!(L.server_m_.empty() && L.server_v_.empty()) && !(L.server_m_.size() == p && L.server_v_.size() == want_v))
      throw std::runtime_error("ledger snapshot: server optimizer state length mismatch");
  }
  L.registered_ = r.vec<int>();
  // every client id in the blob indexes fixed [kCMaxRanks] arrays later (aggregate_locked): a
  // crafted snapshot must not be able to name an id outside [0, client_num)
  auto id = [&](int k) {
    if (k < 0 || k >= c.client_num) throw std::runtime_error("ledger snapshot: client id out of range");
    return k;
  };
  if (static_cast<int64_t>(L.global_.size()) != c.model_size)
    throw std::runtime_error("ledger snapshot: model size mismatch");
  for (int k : L.registered_) id(k);
  for (uint64_t n = r.pod<uint64_t>(), i = 0; i < n; ++i) {
    const int k = id(r.pod<int32_t>());
    L.role_[k] = r.pod<uint32_t>();
  }
  for (uint64_t n = r.pod<uint64_t>(), i = 0; i < n; ++i) {
    LocalUpdate u;
    u.sender = id(r.pod<int32_t>()); u.delta = r.vec<float>(); u.meta.n_samples = r.pod<uint32_t>();
    u.meta.avg_cost = r.pod<float>(); u.arrival = r.pod<uint64_t>();
    if (static_cast<int64_t>(u.delta.size()) != c.model_size)
      throw std::runtime_error("ledger snapshot: update size mismatch");
    L.updates_.emplace(u.sender, std::move(u));
  }
  for (uint64_t n = r.pod<uint64_t>(), i = 0; i < n; ++i) {
    const int c2 = id(r.pod<int32_t>());
    std::map<int, float> row;
    for (uint64_t m = r.pod<uint64_t>(), j = 0; j < m; ++j) {
      const int t = id(r.pod<int32_t>());
      row[t] = r.pod<float>();
    }
    L.scores_[c2] = std::move(row);
  }
  L.arrivals_ = r.pod<uint64_t>(); L.last_loss_ = r.pod<float>();
  for (uint64_t n = r.pod<uint64_t>(), i = 0; i < n; ++i) L.chain_.push_back(read_block(r));
  if (!L.verify_chain()) throw std::runtime_error("snapshot chain fails verification");
  return LP;
}

}  // namespace bflc
