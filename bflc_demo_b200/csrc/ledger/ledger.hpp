// C++ ledger runtime: the committee-consensus state machine of the reference's
// `CommitteePrecompiled` smart contract re-built as a stand-alone, append-only,
// hash-chained block ledger with typed binary payloads.
//
// Reference -> here (FISCO-BCOS/libprecompiled/extension/CommitteePrecompiled.{h,cpp}):
//   N1  #define constants (H:4-19)            -> LedgerConfig (runtime, validated)
//   N2-N4 Model / Meta / LocalUpdate (H:24-107) -> std::vector<float> payload + UpdateMeta
//   N6  7-key table schema (C:31-44)            -> typed members of Ledger
//   N7,N11 ABI selector dispatch (C:46-52,132-167,312-318) -> Ledger::call(Method, ...)
//   N9  GetMid quickselect (C:60-115, buggy)    -> true median (consensus_math.hpp)
//   N12-N17 six handlers (C:168-311)            -> RegisterNode ... QueryAllUpdates
//   N18 Aggregate (C:349-456)                   -> Ledger::aggregate_locked()
//   N19 KV accessors + gas (C:459-512)          -> in-memory state + OpCounters
//   N20 InitGlobalModel (C:321-346)             -> Ledger ctor (epoch = -999, zero model)
//   E1/E2 PBFT replication + table storage      -> Block chain (sha256 prev-hash links),
//                                                  snapshot()/restore(), replica equality
//                                                  check via state_hash()
#pragma once
#include <array>
#include <cstdint>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

namespace bflc {

constexpr int kEpochNotStarted = -999;  // CommitteePrecompiled.cpp:322

struct LedgerConfig {
  int client_num = 20;           // CLIENT_NUM            H:17
  int comm_count = 4;            // COMM_COUNT            H:11
  int aggregate_count = 6;       // AGGREGATE_COUNT       H:13
  int needed_update_count = 10;  // NEEDED_UPDATE_COUNT   H:15
  float learning_rate = 0.001f;  // learning_rate         H:19
  int64_t model_size = 12;       // n_features*n_class + n_class (H:7-8) by default
  int weight_by_score = 0;       // 0 = reference semantics (score filters, n_samples weights)
  int solo = 0;                  // 1 = every client both trains and scores (n = 1 runs)
  uint64_t seed = 0;             // initial committee = seeded permutation (0 -> lowest ids)
  int aggregation = 0;           // AggRule (consensus_math.hpp): 0 FedAvg, 1 median, 2 trimmed mean
  int trim = 1;                  // trimmed mean: updates dropped at each end, 1 <= 2 * trim < aggregate_count
  // server optimizer on the aggregate (consensus_math.hpp ServerOpt / server_step): 0 none, 1 momentum,
  // 2 adam, 3 yogi; the hyperparameters are checked only when it is not none
  int server_opt = 0;
  float server_lr = 1.f;
  float server_beta1 = 0.9f;
  float server_beta2 = 0.99f;
  float server_tau = 1e-3f;
  // differentially private aggregation (consensus_math.hpp DpMode): clip each selected update's model
  // change to L2 norm dp_clip (0 = off), then add Gaussian noise with multiplier dp_noise (0 = clip
  // only; FedAvg only) drawn from dp_seed.  The seed is the secret that makes the noise private: it is
  // neither in the snapshot nor in state_hash (see snapshot()).
  float dp_clip = 0.f;
  float dp_noise = 0.f;
  uint64_t dp_seed = 0;
  int dp_mode() const;   // 0 off, 1 clip, 2 clip + noise
  // adaptive clipping (consensus_math.hpp dp_clip_next): dp_clip_quantile 0 = the fixed clip dp_clip;
  // in (0, 1) the clip starts at dp_clip and tracks that quantile of the selected update norms, at
  // rate dp_clip_lr, from a count noised with dp_count_noise (> dp_noise / 2; 0 in clip-only mode)
  float dp_clip_quantile = 0.f;
  float dp_clip_lr = 0.2f;
  float dp_count_noise = 0.f;
  bool dp_adaptive() const { return dp_clip_quantile != 0.f; }
  int dp_kernel_mode() const;   // the consensus kernel's / block record's mode: 0 .. 4 (DpMode)
  // returns "" when the invariant COMM <= AGG <= NEEDED <= CLIENT - COMM holds
  std::string validate() const;
};

// xi_i for coordinates first .. first + n - 1 of round `epoch` (consensus_math.hpp dp_gauss4)
void dp_gauss_fill(uint64_t seed, uint32_t epoch, uint64_t first, float* out, size_t n);

enum class Status : int {
  OK = 0,
  NOT_STARTED = 1,
  STALE_EPOCH = 2,       // C:225, C:268
  DUPLICATE = 3,         // C:232
  QUOTA_FULL = 4,        // C:239
  NOT_COMMITTEE = 5,     // C:274
  UNKNOWN_CLIENT = 6,
  BAD_PAYLOAD = 7,
  AGGREGATED = 8,        // OK + this call closed the round (C:296-297)
  NOT_TRAINER = 9,       // committee members do not upload in their committee round (M:259-263)
  NOT_READY = 10,        // scores before the update quota is filled
};
const char* status_name(Status s);

struct UpdateMeta {
  uint32_t n_samples = 0;  // H:56
  float avg_cost = 0.f;    // H:57
};

struct LocalUpdate {
  int sender = -1;
  std::vector<float> delta;  // (w_old - w_new) / lr, main.py:153-154
  UpdateMeta meta;
  uint64_t arrival = 0;      // admission order (tx order in the reference)
};

using Hash256 = std::array<uint8_t, 32>;
Hash256 sha256(const void* data, size_t n);
std::string hex(const Hash256& h);

struct Block {
  uint64_t index = 0;
  int epoch = 0;  // the round this block closes
  Hash256 prev_hash{};
  Hash256 hash{};
  std::vector<uint32_t> role_before, role_after;
  std::vector<int> admitted;             // in admission order
  std::vector<int> committee;            // members that scored
  std::vector<std::vector<float>> scores;  // [committee index][admitted index]
  std::vector<float> median;             // per admitted
  std::vector<int> selected;             // aggregated trainers (rank order)
  std::vector<float> weight;             // per selected
  float global_loss = 0.f;
  Hash256 model_hash{};                  // sha256 of the new global model (host path)
  uint64_t device_digest = 0;            // digest computed by the consensus kernel (GPU path)
  uint8_t from_device = 0;
};

struct OpCounters {  // replaces the gas meter (C:143,151,468-469,...) as plain metrics
  uint64_t calls = 0, register_ok = 0, uploads_ok = 0, uploads_rejected = 0, scores_ok = 0,
           scores_rejected = 0, aggregations = 0, queries = 0;
};

// The contract's method table (reference: six Solidity signatures -> 4-byte selectors,
// CommitteePrecompiled.cpp:46-52,122-130; interface stub python-sdk/contracts/
// CommitteePrecompiled.sol:3-10).  Signatures are kept verbatim so external tooling written
// against the reference ABI can address the same methods by name.
enum class Method : int {
  RegisterNode = 0,
  QueryState = 1,
  QueryGlobalModel = 2,
  UploadLocalUpdate = 3,
  UploadScores = 4,
  QueryAllUpdates = 5,
  Unknown = -1,  // C:312-318: unknown selector -> error
};
struct MethodInfo {
  Method id;
  const char* signature;  // e.g. "UploadLocalUpdate(string,int256)"
  bool is_view;           // client.call (view) vs sendRawTransactionGetReceipt (tx)
};
const MethodInfo* method_table(int* n);
Method method_from_signature(const std::string& signature_or_name);

class Ledger {
 public:
  explicit Ledger(const LedgerConfig& cfg);

  // --- the six contract methods (S:3-10); `client` replaces the tx origin address ---
  Status RegisterNode(int client);
  // returns role bits (unknown client reported as trainer, C:197-200) and the epoch
  std::pair<uint32_t, int> QueryState(int client);
  std::pair<std::vector<float>, int> QueryGlobalModel();
  Status UploadLocalUpdate(int client, const std::vector<float>& delta, UpdateMeta meta, int ep);
  Status UploadScores(int client, int ep, const std::map<int, float>& scores);
  // empty until needed_update_count updates are in (C:304-307)
  std::vector<LocalUpdate> QueryAllUpdates();

  // --- GPU path: adopt a round decided by the device consensus kernel, after re-executing
  //     the election from its raw score rows (state-machine-replication check) ---
  struct DeviceRound {
    int epoch = 0;
    std::vector<uint32_t> role_before, role_after;
    std::vector<std::vector<float>> score_rows;  // [rank][rank]
    std::vector<uint32_t> scored_mask;
    std::vector<uint32_t> n_samples;
    std::vector<float> avg_cost;
    uint32_t admitted_mask = 0, selected_mask = 0;
    float global_loss = 0.f;
    uint64_t model_digest = 0;
    int weight_by_score = 0;
    uint32_t agg = 0;  // the record's aggregation word, agg_word(rule, trim, server_opt, dp mode)
    // adaptive clipping: the round's DpClipRecord (clip C_t, noised count b~, selected count)
    int has_clip = 0;
    float clip = 0.f, count = 0.f;
    uint32_t n_sel = 0;
  };
  // returns "" on success, else the first mismatch
  std::string AppendDeviceRound(const DeviceRound& r);
  // start the chain directly at epoch 0 with the given roles (device bootstrap)
  void Bootstrap(const std::vector<uint32_t>& roles);

  // --- introspection / persistence ---
  int epoch() const;
  const LedgerConfig& config() const { return cfg_; }
  std::vector<uint32_t> roles() const;
  std::vector<Block> blocks() const;
  size_t n_blocks() const;
  OpCounters counters() const;
  std::vector<std::string> drain_log();
  float last_global_loss() const;
  Hash256 state_hash() const;      // replicas must agree on this after every block
  bool verify_chain() const;       // recompute every block hash + prev links
  std::string snapshot() const;    // binary checkpoint (blocks + live state)
  // dp_seed: the DP noise seed of the restored ledger (a snapshot never holds it)
  static std::unique_ptr<Ledger> restore(const std::string& blob, uint64_t dp_seed = 0);
  int update_count() const;
  int score_count() const;
  // host-path server optimizer state {m, v}: empty until the first host aggregation (device mode
  // keeps it in HBM instead), v empty for momentum
  std::pair<std::vector<float>, std::vector<float>> server_state() const;
  // adaptive clipping: the clip of the next round, and (C_t, b~, n_sel) of the last aggregated round
  float dp_clip_now() const;
  struct ClipStep {
    float clip = 0.f, count = 0.f;
    int n_sel = 0;
  };
  ClipStep last_clip_step() const;

 private:
  void aggregate_locked();
  void append_block_locked(Block&& b);
  Hash256 hash_block(const Block& b) const;
  void log(std::string s);

  LedgerConfig cfg_;
  mutable std::mutex mu_;
  int epoch_ = kEpochNotStarted;
  std::vector<float> global_;
  std::vector<int> registered_;            // registration order
  std::map<int, uint32_t> role_;           // client -> RoleBits
  std::map<int, LocalUpdate> updates_;     // admitted this round
  std::map<int, std::map<int, float>> scores_;  // committee -> (trainer -> score)
  uint64_t arrivals_ = 0;
  std::vector<Block> chain_;
  OpCounters ctr_;
  std::vector<std::string> log_;
  float last_loss_ = 0.f;
  std::vector<float> server_m_, server_v_;  // allocated lazily by aggregate_locked
  float clip_now_ = 0.f;                    // adaptive clipping: C_t (dp_clip at genesis)
  ClipStep last_clip_;
};

}  // namespace bflc
