// The three communication-bound steps of a committee-consensus round as sm_90a kernels
// that talk to peer GPUs themselves (ld/st/atom on peer-mapped HBM over NVLink 4 /
// NVSwitch, optional NVLS multimem stores) -- no NCCL call on these paths.
//
//   fed_plan_round          X2  QueryState        -> local read of the HBM ledger page
//   fed_upload              X4  UploadLocalUpdate -> publish + release flag on every peer
//   (validation GEMM)       X5  QueryAllUpdates   -> TMA pulls of peers' weights (gemm_sm100.cu)
//   fed_consensus_aggregate X6  UploadScores      -> score row pushed to every replica
//                           X7  Aggregate         -> in-kernel median/top-K + FedAvg (or a robust
//                                                    median / trimmed mean) over P2P
//                           X3  QueryGlobalModel  -> result written straight into the next
//                                                    round's training buffers
// (X-numbers: SURVEY.md 2.7b; reference semantics: CommitteePrecompiled.cpp:168-456.)
//
// Synchronisation is by monotonically increasing, epoch-tagged 32-bit flags written with
// st.release.sys and polled with ld.acquire.sys; nothing is ever reset, so there is no
// reuse race when committee membership changes between rounds.
#include <cuda_bf16.h>

#include "bflc_kernels.h"
#include "consensus_math.hpp"
#include "epi_common.cuh"
#include "fed_admit.cuh"
#include "launch.cuh"
#include "sm100_ptx.cuh"

namespace bflc {

namespace {

constexpr int kFedThreads = 256;

template <typename T>
__device__ __forceinline__ T* at(char* base, long long off) {
  return reinterpret_cast<T*>(base + off);
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}

// ------------------------------------------------------------------ plan
struct PlanLayers {
  PlanLayer l[kMaxPlanLayers];
  int n;
  int steps_per_round;
  int staged;  // 1: validation B operands are the local staging slots filled by k_pull
  // fp8 MLP: candidates are Mx8MlpLayout blobs -- local staging slot z, or (direct) the trainer's
  // upload blob at heap offset upq_off[parity]
  int use_blob;
  uint8_t* stage_blob; long long blob_bytes; long long upq_off[2];
  // staged: candidate z's fp32 parameters (k_pull's stage_master, at least the bias ranges) at
  // stage_master + z * n_params -- the validation biases.  Null: the biases are read from the
  // candidate's upload buffer, which needs its rank here (every trainer awaited, or direct mode).
  const float* stage_master;
};

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void stamp(RoundPlan* plan, int slot) {
  atomicMax(&plan->t_stamp[slot], globaltimer_ns());
}

__global__ void k_plan(FedArgs f, PlanLayers layers) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  char* me = f.peers.base[f.rank];
  const RoundState* st = at<RoundState>(me, f.lay.state_off);
  RoundPlan* plan = at<RoundPlan>(me, f.lay.plan_off);
  for (int i = 0; i < 8; ++i) plan->t_stamp[i] = 0;
  plan->t_stamp[STAMP_PLAN] = globaltimer_ns();
  uint32_t* flags = at<uint32_t>(me, f.lay.flags_off);
  const uint32_t epoch = st->epoch;
  const uint32_t par = epoch & 1u;
  // Buffers of parity `par` were last read by peers while aggregating epoch - 2.
  if (epoch >= 2) {
    for (int r = 0; r < f.n_ranks; ++r) ptx::wait_flag_ge(flags + FLAG_DONE + r, epoch - 1);
  }
  plan->is_trainer = (st->role[f.rank] & ROLE_TRAINER) ? 1 : 0;
  plan->is_comm = (st->role[f.rank] & ROLE_COMM) ? 1 : 0;
  plan->parity = par;
  int n_cand = 0;
  for (int r = 0; r < f.n_ranks; ++r)
    if (st->role[r] & ROLE_TRAINER) plan->cand_rank[n_cand++] = r;
  if (admit::first_k(st)) {
    // first-K-wins: candidate slot z is whoever takes ticket z this round -- resolved by the
    // consumers of the slot (k_pull*, k_consensus), not here
    n_cand = static_cast<int>(st->n_needed);
    for (int z = 0; z < kMaxRanks; ++z) plan->cand_rank[z] = -1;
  }
  plan->n_cand = n_cand;
  for (int l = 0; l < layers.n; ++l) {
    GemmDynamic& d = plan->dyn[l];
    d.active_batches = plan->is_comm ? n_cand : 0;
    d.wait_value = epoch + 1;
    for (int z = 0; z < kMaxRanks; ++z) {
      const int t = (z < n_cand && plan->cand_rank[z] >= 0) ? plan->cand_rank[z] : 0;
      // tensor-map table: staged -> [layer][slot] over local staging; direct -> [layer][parity]
      // [rank] over the trainers' upload buffers (TMA pulls across NVLink)
      d.map_index[z] = layers.staged ? (l * kMaxRanks + z)
                                     : ((l * 2 + static_cast<int>(par)) * kMaxRanks + t);
      // staged with stage_master: slot z's own fp32 copy (in first-K mode slot z's trainer is only
      // known once it takes a ticket, so t would be rank 0 here)
      const float* params = layers.staged && layers.stage_master != nullptr
                                ? layers.stage_master + static_cast<long long>(z) * f.lay.n_params
                                : at<float>(f.peers.base[t], f.lay.upload_master_off[par]);
      d.bias[z] = layers.l[l].use_bias ? params + layers.l[l].bias_off : nullptr;
      d.wait_flag[z] = layers.staged ? nullptr : flags + FLAG_TRAINED + t;
    }
  }
  for (int z = 0; z < kMaxRanks; ++z) {
    plan->correct[z] = 0;
    const int t = (z < n_cand && plan->cand_rank[z] >= 0) ? plan->cand_rank[z] : f.rank;
    plan->cand_blob[z] = !layers.use_blob ? nullptr
                         : layers.staged  ? layers.stage_blob + z * layers.blob_bytes
                                          : reinterpret_cast<const uint8_t*>(f.peers.base[t]) + layers.upq_off[par];
  }
  plan->loss_sum = 0.f;
  plan->train_correct = 0;
  plan->upload_blocks_done = 0;
  plan->consensus_blocks_done = 0;
  plan->digest_acc = 0ull;
  plan->step_barrier = 0u;
  plan->round_seq = plan->round_seq + 1u;   // input-pipeline generation (matches k_cast_chunks' ready[])
  plan->opt_step = plan->opt_total;
  if (plan->is_trainer) plan->opt_total += layers.steps_per_round;
}

// ------------------------------------------------------------------ upload
__global__ void __launch_bounds__(kFedThreads)
k_upload(FedArgs f, int n_samples, int n_loss_terms, int byz_mode, float byz_scale, int straggle_us) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  char* me = f.peers.base[f.rank];
  const RoundState* st = at<RoundState>(me, f.lay.state_off);
  RoundPlan* plan = at<RoundPlan>(me, f.lay.plan_off);
  if (!(st->role[f.rank] & ROLE_TRAINER)) return;
  if (blockIdx.x == 0 && threadIdx.x == 0) stamp(plan, STAMP_UPLOAD_BEGIN);
  const uint32_t epoch = st->epoch;
  const uint32_t par = epoch & 1u;
  const float4* wm = at<const float4>(me, f.lay.work_master_off);
  const float4* gm = at<const float4>(me, f.lay.global_off);
  float4* um = at<float4>(me, f.lay.upload_master_off[par]);
  uint2* us = at<uint2>(me, f.lay.upload_shadow_off[par]);
  const long long nv = f.lay.n_params / 4;
  const long long tid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = tid; i < nv; i += stride) {
    float4 w = wm[i];
    if (byz_mode == 1) {
      // Byzantine client: upload global - scale * (honest step) instead of the honest model
      const float4 g = gm[i];
      w.x = g.x - byz_scale * (w.x - g.x);
      w.y = g.y - byz_scale * (w.y - g.y);
      w.z = g.z - byz_scale * (w.z - g.z);
      w.w = g.w - byz_scale * (w.w - g.w);
    }
    um[i] = w;
    us[i] = make_uint2(pack_bf16x2(w.x, w.y), pack_bf16x2(w.z, w.w));
  }
  // publish: the block barrier orders every thread's writes before thread 0's system-scope
  // fence (release patterns are cumulative), the last block to arrive raises the flags
  __syncthreads();
  __shared__ bool last;
  if (threadIdx.x == 0) {
    __threadfence_system();
    const unsigned done = atomicAdd(&plan->upload_blocks_done, 1u);
    last = (done == gridDim.x - 1);
  }
  __syncthreads();
  if (!last) return;
  __threadfence_system();
  // first-K-wins admission: one ticket per trainer and round; late tickets publish nothing
  __shared__ int ticket;
  if (threadIdx.x == 0) {
    admit::straggle(straggle_us);
    ticket = admit::first_k(st) ? admit::take_ticket(&admit::page(f.peers.base[0], f.lay, par)->ticket, epoch) : 0;
    if (ticket >= static_cast<int>(st->n_needed) && admit::first_k(st)) ticket = -1;
  }
  __syncthreads();
  if (ticket >= 0 && threadIdx.x < f.n_ranks) {
    const int r = threadIdx.x;
    UploadMeta* meta = at<UploadMeta>(f.peers.base[r], f.lay.meta_off) + par * kMaxRanks + f.rank;
    UploadMeta m;
    m.n_samples = static_cast<uint32_t>(n_samples);
    m.avg_cost = plan->loss_sum / static_cast<float>(n_loss_terms > 0 ? n_loss_terms : 1);
    *meta = m;
    __threadfence_system();
    if (admit::first_k(st))
      ptx::st_release_sys(&admit::page(f.peers.base[r], f.lay, par)->slot[ticket],
                          ((epoch + 1u) << 8) | static_cast<uint32_t>(f.rank));
    ptx::st_release_sys(at<uint32_t>(f.peers.base[r], f.lay.flags_off) + FLAG_TRAINED + f.rank,
                        epoch + 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) stamp(plan, STAMP_UPLOAD_END);
}

// --------------------------------------------------------------- consensus
struct ConsShared {
  ConsensusIn<kMaxRanks> in;
  ConsensusOut<kMaxRanks> out;
  int sel_rank[kMaxRanks];
  float sel_w[kMaxRanks];
  int n_sel;
};

__device__ __forceinline__ unsigned long long digest_term(float v, long long idx) {
  // order-independent (sum of per-element terms) so any reduction schedule gives the same
  // digest; odd multiplier keeps every bit of the float significant.
  return static_cast<unsigned long long>(__float_as_uint(v)) *
         (static_cast<unsigned long long>(2 * idx + 1) * 0x9E3779B97F4A7C15ull);
}

// What thread 0 of every consensus block derives from the norm partials (kDp != DP_OFF only).
struct DpShared {
  float s[kMaxRanks];          // clip factor of selected update k (ascending rank order)
  float norm[kMaxRanks];       // n_t by trainer rank (NaN: not admitted)
  float scale[kMaxRanks];      // s_t by trainer rank (NaN: not admitted)
  float sigma;
  uint32_t clipped;            // bit k: selected update k is clipped (s_k != 1)
};

// kRobust: step (d) is the coordinate-wise trimmed mean / median of the selected uploads
// (consensus_math.hpp robust_combine) instead of FedAvg; agg = agg_word(rule, trim, kServerOpt, kDp).
// kServerOpt (ServerOpt): the new global model is server_step(global, combined) instead of the
// combined value itself, with this rank's optimizer state (so) in local HBM; 0 = none.
// kDp (DpMode): each selected upload is clipped to L2 distance dp.clip from the global model before
// the rule combines it (norms from the DpPage partials of k_update_norms), and with DP_NOISE the
// FedAvg aggregate gets Gaussian noise before the server step; DP_OFF is the k_consensus kernel.
template <bool kRobust, int kServerOpt, int kDp>
__device__ __forceinline__ void consensus_body(FedArgs f, int n_val, int weight_by_score, int two_shot, int use_mc,
                                               uint32_t* host_mirror, uint32_t* bump_seq, uint32_t agg,
                                               ServerOptArgs so, DpArgs dp, DpShared* dsh) {
  __shared__ ConsShared sh;
  __shared__ bool last;
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  char* me = f.peers.base[f.rank];
  RoundState* st = at<RoundState>(me, f.lay.state_off);
  RoundPlan* plan = at<RoundPlan>(me, f.lay.plan_off);
  uint32_t* flags = at<uint32_t>(me, f.lay.flags_off);
  const uint32_t epoch = st->epoch;
  const uint32_t par = epoch & 1u;
  const int n = f.n_ranks;
  const bool i_am_comm = (st->role[f.rank] & ROLE_COMM) != 0;
  if (blockIdx.x == 0 && threadIdx.x == 0) stamp(plan, STAMP_CONS_BEGIN);

  // first-K-wins: candidate slot z -> admitted trainer (every block resolves all K slots; the
  // acquire also makes those trainers' uploads readable)
  const bool fk = admit::first_k(st);
  __shared__ int cand_of[kMaxRanks];
  __shared__ uint32_t adm_mask;
  if (threadIdx.x == 0) {
    uint32_t m = 0;
    for (int z = 0; z < plan->n_cand; ++z) {
      cand_of[z] = fk ? admit::wait_slot(admit::page(me, f.lay, par), z, epoch) : plan->cand_rank[z];
      m |= 1u << cand_of[z];
    }
    adm_mask = m;
  }
  __syncthreads();

  // (a) committee: push my score row into every replica's ledger page, then release.
  if (blockIdx.x == 0 && i_am_comm) {
    if (threadIdx.x < n) {
      const int r = threadIdx.x;  // destination replica
      float* row = at<float>(f.peers.base[r], f.lay.scores_off) +
                   (par * kMaxRanks + f.rank) * kMaxRanks;
      for (int z = 0; z < plan->n_cand; ++z)
        row[cand_of[z]] =
            static_cast<float>(plan->correct[z]) / static_cast<float>(n_val > 0 ? n_val : 1);
      // the row was written by THIS lane: the sys-scope release store below orders it, no
      // separate membar.sys (which also waited for every other outstanding write of the SM)
      ptx::st_release_sys(at<uint32_t>(f.peers.base[r], f.lay.flags_off) + FLAG_SCORED + f.rank,
                          epoch + 1);
    }
  }

  // (b) every block: wait for all committee rows and all trainer uploads (local polls)
  if (threadIdx.x < n) {
    const int r = threadIdx.x;
    if (st->role[r] & ROLE_COMM) ptx::wait_flag_ge(flags + FLAG_SCORED + r, epoch + 1);
    // every admitted trainer's upload (first-K-wins: only the K ticket holders -- a straggler or
    // a dead trainer beyond them is not waited for)
    if ((st->role[r] & ROLE_TRAINER) && ((adm_mask >> r) & 1u)) ptx::wait_flag_ge(flags + FLAG_TRAINED + r, epoch + 1);
  }
  __syncthreads();
  if (blockIdx.x == 0 && threadIdx.x == 0) stamp(plan, STAMP_CONS_SCORED);

  // (c) consensus math, redundantly per block (tiny), identical on every rank.  The 64 score
  //     words and 16 meta words are fetched by 80 threads at once (a single thread paid one L2
  //     round trip per word: ~12 us of the old 25 us kernel), then thread 0 runs the decision
  //     procedure out of shared memory.
  {
    ConsensusIn<kMaxRanks>& in = sh.in;
    const float* rows = at<float>(me, f.lay.scores_off) + par * kMaxRanks * kMaxRanks;
    const UploadMeta* meta = at<UploadMeta>(me, f.lay.meta_off) + par * kMaxRanks;
    const int i = threadIdx.x;
    if (i < kMaxRanks * kMaxRanks) {
      const int r = i / kMaxRanks, t = i % kMaxRanks;
      const bool ok = r < n && t < n && (st->role[r] & ROLE_COMM) && (st->role[t] & ROLE_TRAINER) &&
                      ((adm_mask >> t) & 1u);
      in.scored[r][t] = ok ? 1 : 0;
      in.score[r][t] =
          ok ? __uint_as_float(ptx::ld_relaxed_sys(reinterpret_cast<const uint32_t*>(rows + r * kMaxRanks + t))) : 0.f;
    } else if (i < kMaxRanks * kMaxRanks + kMaxRanks) {
      const int r = i - kMaxRanks * kMaxRanks;
      in.role[r] = r < n ? st->role[r] : 0u;
      in.admitted[r] = (r < n && (st->role[r] & ROLE_TRAINER) && ((adm_mask >> r) & 1u)) ? 1 : 0;
      in.n_samples[r] = r < n ? ptx::ld_relaxed_sys(&meta[r].n_samples) : 0u;
      in.avg_cost[r] =
          r < n ? __uint_as_float(ptx::ld_relaxed_sys(reinterpret_cast<const uint32_t*>(&meta[r].avg_cost))) : 0.f;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    ConsensusIn<kMaxRanks>& in = sh.in;
    in.n_ranks = n;
    in.n_comm = static_cast<int>(st->n_comm);
    in.n_aggregate = static_cast<int>(st->n_aggregate);
    in.weight_by_score = weight_by_score;
    run_consensus<kMaxRanks>(in, sh.out);
    int k = 0;
    for (int r = 0; r < n; ++r)  // ascending rank = the fixed reduction order
      if (sh.out.selected[r]) {
        sh.sel_rank[k] = r;
        sh.sel_w[k] = sh.out.weight[r];
        ++k;
      }
    sh.n_sel = k;
  }
  __syncthreads();
  if constexpr (kDp != DP_OFF) {
    // every rank's norm partials of this epoch, added in rank order: identical on every replica
    if (threadIdx.x < n) ptx::wait_flag_ge(flags + FLAG_NORM + threadIdx.x, epoch + 1);
    __syncthreads();
    if (threadIdx.x == 0) {
      const volatile double* part = at<const double>(me, dp.off + offsetof(DpPage, partial)) + par * kMaxRanks * kMaxRanks;
      for (int t = 0; t < kMaxRanks; ++t) {
        float nrm = __uint_as_float(0x7FC00000u), sc = nrm;
        if (sh.in.admitted[t]) {
          double sum = 0.0;
          for (int q = 0; q < n; ++q) sum += part[q * kMaxRanks + t];
          nrm = dp_norm(sum);
          sc = dp_scale(nrm, dp.clip);
        }
        dsh->norm[t] = nrm;
        dsh->scale[t] = sc;
      }
      uint32_t clipped = 0, wmax = 0;
      for (int k = 0; k < sh.n_sel; ++k) {
        const float sc = dsh->scale[sh.sel_rank[k]];
        dsh->s[k] = sc;
        if (dp_bits(sc) != 0x3F800000u) clipped |= 1u << k;
        const uint32_t wb = dp_bits(sh.sel_w[k]);   // weights are >= 0: the bit patterns order them
        wmax = wb > wmax ? wb : wmax;
      }
      dsh->clipped = clipped;
      dsh->sigma = kDp == DP_NOISE && sh.n_sel > 0 ? so_mul(so_mul(dp.noise, dp.clip), dp_float(wmax)) : 0.f;
    }
    __syncthreads();
  }

  // (d) FedAvg: new_global = sum_k w_k * upload_k   (reference C:373-414, with
  //     delta = (w_old - w_new)/lr this is exactly global -= lr * weighted-mean(delta)).
  //     Robust: new_global = per-coordinate trimmed mean of the selected uploads, unweighted.
  const int n_sel = sh.n_sel;
  const int trim = agg_trim(static_cast<int>(agg & 0xFFu), static_cast<int>((agg >> 8) & 0xFFu), n_sel);
  const float4* src[kMaxRanks];
  float w[kMaxRanks];
#pragma unroll
  for (int k = 0; k < kMaxRanks; ++k) {
    const int r = k < n_sel ? sh.sel_rank[k] : f.rank;
    src[k] = at<const float4>(f.peers.base[r], f.lay.upload_master_off[par]);
    w[k] = k < n_sel ? sh.sel_w[k] : 0.f;
  }
  const long long nv = f.lay.n_params / 4;
  long long lo = 0, hi = nv;
  if (two_shot) {  // each rank reduces only its own slice, then publishes it to every peer
    long long per = (nv + n - 1) / n;
    per += per & 1;   // even slices: two neighbouring lanes pair their bf16 halves into one 16-byte store
    lo = per * f.rank;
    hi = lo + per < nv ? lo + per : nv;
    if (lo > nv) lo = nv;
  }
  float4* g_f32 = at<float4>(me, f.lay.global_off);
  uint2* g_b16 = at<uint2>(me, f.lay.global_shadow_off);
  float4* w_f32 = at<float4>(me, f.lay.work_master_off);
  uint2* w_b16 = at<uint2>(me, f.lay.work_shadow_off);
  const bool mc = two_shot && use_mc && f.peers.mc_base != nullptr;
  float4* s_m = at<float4>(me, so.m_off);   // server optimizer state (kServerOpt != 0 only)
  float4* s_v = at<float4>(me, so.v_off);
  unsigned long long dig = 0ull;
  const long long tid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = lo + tid; i < hi; i += stride) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (n_sel == 0) {
      acc = g_f32[i];  // nothing admitted: the global model is unchanged
    } else {
      float4 v[kMaxRanks];
#pragma unroll
      for (int k = 0; k < kMaxRanks; ++k)
        if (k < n_sel) v[k] = ptx::ld_peer_f4(src[k] + i);  // all peer loads in flight first
      if constexpr (kDp != DP_OFF) {
        // clip while loading: an unclipped update stays bit for bit the upload
        const float4 g = g_f32[i];
        const uint32_t clipped = dsh->clipped;
#pragma unroll
        for (int k = 0; k < kMaxRanks; ++k)
          if (k < n_sel && ((clipped >> k) & 1u)) {
            const float s = dsh->s[k];
            v[k].x = dp_clip_value(g.x, v[k].x, s);
            v[k].y = dp_clip_value(g.y, v[k].y, s);
            v[k].z = dp_clip_value(g.z, v[k].z, s);
            v[k].w = dp_clip_value(g.w, v[k].w, s);
          }
      }
      if constexpr (kRobust) {
        float c[kMaxRanks];
#pragma unroll
        for (int k = 0; k < kMaxRanks; ++k) c[k] = v[k].x;
        acc.x = robust_combine<kMaxRanks>(c, n_sel, trim);
#pragma unroll
        for (int k = 0; k < kMaxRanks; ++k) c[k] = v[k].y;
        acc.y = robust_combine<kMaxRanks>(c, n_sel, trim);
#pragma unroll
        for (int k = 0; k < kMaxRanks; ++k) c[k] = v[k].z;
        acc.z = robust_combine<kMaxRanks>(c, n_sel, trim);
#pragma unroll
        for (int k = 0; k < kMaxRanks; ++k) c[k] = v[k].w;
        acc.w = robust_combine<kMaxRanks>(c, n_sel, trim);
      } else {
#pragma unroll
        for (int k = 0; k < kMaxRanks; ++k)
          if (k < n_sel) {
            acc.x = fmaf(w[k], v[k].x, acc.x);
            acc.y = fmaf(w[k], v[k].y, acc.y);
            acc.z = fmaf(w[k], v[k].z, acc.z);
            acc.w = fmaf(w[k], v[k].w, acc.w);
          }
      }
      if constexpr (kDp == DP_NOISE) {
        float z[4];
        dp_gauss4(dp.seed, epoch, static_cast<uint64_t>(i), z, kDpSite);
        const float sigma = dsh->sigma;
        acc.x = so_add(acc.x, so_mul(sigma, z[0]));
        acc.y = so_add(acc.y, so_mul(sigma, z[1]));
        acc.z = so_add(acc.z, so_mul(sigma, z[2]));
        acc.w = so_add(acc.w, so_mul(sigma, z[3]));
      }
      if constexpr (kServerOpt != SOPT_NONE) {
        // the step from the (identical on every rank) local global model; each rank owns the state
        // of the coordinates it reduces, so two-shot slices keep it local as well
        const ServerOptParams p{so.lr, so.b1, so.b2, so.c1, so.c2, so.tau};
        const float4 g = g_f32[i];
        float4 m = s_m[i];
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if constexpr (kServerOpt != SOPT_MOMENTUM) v = s_v[i];
        acc.x = server_step(kServerOpt, g.x, acc.x, m.x, v.x, p);
        acc.y = server_step(kServerOpt, g.y, acc.y, m.y, v.y, p);
        acc.z = server_step(kServerOpt, g.z, acc.z, m.z, v.z, p);
        acc.w = server_step(kServerOpt, g.w, acc.w, m.w, v.w, p);
        s_m[i] = m;
        if constexpr (kServerOpt != SOPT_MOMENTUM) s_v[i] = v;
      }
    }
    dig += digest_term(acc.x, 4 * i) + digest_term(acc.y, 4 * i + 1) +
           digest_term(acc.z, 4 * i + 2) + digest_term(acc.w, 4 * i + 3);
    const uint2 b = make_uint2(pack_bf16x2(acc.x, acc.y), pack_bf16x2(acc.z, acc.w));
    if (!two_shot) {
      g_f32[i] = acc; g_b16[i] = b; w_f32[i] = acc; w_b16[i] = b;
    } else if (mc) {
      // one NVLS store per destination buffer lands in all replicas
      ptx::multimem_st_f4(at<float4>(f.peers.mc_base, f.lay.global_off) + i, acc);
      ptx::multimem_st_f4(at<float4>(f.peers.mc_base, f.lay.work_master_off) + i, acc);
      // bf16 copies: the even lane of each lane pair takes its neighbour's 8 bytes and issues ONE
      // 16-byte multimem store per buffer (slices are even, so pairs are never split); before,
      // these were 2 x n_ranks 8-byte P2P stores per thread -- 80 % of the publish traffic
      const unsigned am = __activemask();
      const uint32_t ox = __shfl_down_sync(am, b.x, 1), oy = __shfl_down_sync(am, b.y, 1);
      if ((i & 1) == 0) {
        const float4 pk = make_float4(__uint_as_float(b.x), __uint_as_float(b.y), __uint_as_float(ox),
                                      __uint_as_float(oy));
        ptx::multimem_st_f4(at<float4>(f.peers.mc_base, f.lay.global_shadow_off) + (i >> 1), pk);
        ptx::multimem_st_f4(at<float4>(f.peers.mc_base, f.lay.work_shadow_off) + (i >> 1), pk);
      }
    } else {
      for (int r = 0; r < n; ++r) {
        char* pb = f.peers.base[r];
        at<float4>(pb, f.lay.global_off)[i] = acc;
        at<uint2>(pb, f.lay.global_shadow_off)[i] = b;
        at<float4>(pb, f.lay.work_master_off)[i] = acc;
        at<uint2>(pb, f.lay.work_shadow_off)[i] = b;
      }
    }
  }
  // block-level digest reduce
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) dig += __shfl_xor_sync(0xffffffffu, dig, off);
  if ((threadIdx.x & 31) == 0 && dig) atomicAdd(&plan->digest_acc, dig);

  // (e) last block: commit the round
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    const unsigned done = atomicAdd(&plan->consensus_blocks_done, 1u);
    last = (done == gridDim.x - 1);
  }
  __syncthreads();
  if (!last) return;
  __threadfence_system();

  if (two_shot) {
    // publish my slice (+ its digest) and wait for everyone else's
    if (threadIdx.x < n) {
      const int r = threadIdx.x;
      unsigned long long* slot =
          reinterpret_cast<unsigned long long*>(at<float>(f.peers.base[r], f.lay.scores_off) +
                                                2 * kMaxRanks * kMaxRanks) +
          par * kMaxRanks + f.rank;
      *slot = *reinterpret_cast<volatile unsigned long long*>(&plan->digest_acc);
      __threadfence_system();
      ptx::st_release_sys(at<uint32_t>(f.peers.base[r], f.lay.flags_off) + FLAG_SLICE + f.rank,
                          epoch + 1);
    }
    __syncthreads();
    if (threadIdx.x < n) ptx::wait_flag_ge(flags + FLAG_SLICE + threadIdx.x, epoch + 1);
    __syncthreads();
  }

  if (threadIdx.x == 0) {
    unsigned long long digest = 0ull;
    if (two_shot) {
      const unsigned long long* slots =
          reinterpret_cast<const unsigned long long*>(at<float>(me, f.lay.scores_off) +
                                                      2 * kMaxRanks * kMaxRanks) +
          par * kMaxRanks;
      for (int r = 0; r < n; ++r)
        digest += *reinterpret_cast<const volatile unsigned long long*>(slots + r);
    } else {
      digest = *reinterpret_cast<volatile unsigned long long*>(&plan->digest_acc);
    }
    const ConsensusIn<kMaxRanks>& in = sh.in;
    const ConsensusOut<kMaxRanks>& out = sh.out;
    // append the block record (drained by the host ledger)
    BlockRecord* rec =
        at<BlockRecord>(me, f.lay.ring_off) + (epoch % static_cast<uint32_t>(f.lay.ring_slots));
    rec->epoch = epoch;
    rec->n_ranks = static_cast<uint32_t>(n);
    rec->n_comm = st->n_comm;
    rec->n_aggregate = st->n_aggregate;
    uint32_t adm = 0, sel = 0;
    for (int r = 0; r < kMaxRanks; ++r) {
      rec->role_before[r] = in.role[r];
      rec->role_after[r] = r < n ? out.role_after[r] : 0u;
      uint32_t m = 0;
      for (int t = 0; t < kMaxRanks; ++t) {
        rec->score_rows[r][t] = in.score[r][t];
        if (in.scored[r][t]) m |= 1u << t;
      }
      rec->scored_mask[r] = m;
      rec->median[r] = r < n ? out.median[r] : 0.f;
      rec->n_samples[r] = in.n_samples[r];
      rec->avg_cost[r] = in.avg_cost[r];
      rec->weight[r] = r < n ? out.weight[r] : 0.f;
      if (in.admitted[r]) adm |= 1u << r;
      if (r < n && out.selected[r]) sel |= 1u << r;
    }
    rec->admitted_mask = adm;
    rec->selected_mask = sel;
    rec->global_loss = out.global_loss;
    rec->weight_by_score = static_cast<uint32_t>(weight_by_score);
    rec->model_digest = digest;
    rec->agg = agg;
    __threadfence();
    rec->seq = epoch + 1;
    // advance the ledger page: re-election, epoch++
    for (int r = 0; r < n; ++r) {
      st->role[r] = out.role_after[r];
      st->last_median[r] = out.median[r];
    }
    st->selected_mask = sel;
    st->global_loss = out.global_loss;
    st->model_digest = digest;
    st->blocks_appended = st->blocks_appended + 1;
    st->epoch = epoch + 1;
    if constexpr (kDp != DP_OFF) {   // this round's norms and clip factors, for the engines to read back
      DpPage* page = at<DpPage>(me, dp.off);
      for (int t = 0; t < kMaxRanks; ++t) {
        page->norm[t] = dsh->norm[t];
        page->scale[t] = dsh->scale[t];
      }
      page->sigma = dsh->sigma;
      page->epoch = epoch + 1;
    }
    __threadfence_system();
  }
  __syncthreads();
  // input pipeline: every reader of this round's tag (input kernel, trainer) is done -- count
  // the round so the next one expects the next tag
  if (bump_seq != nullptr && threadIdx.x == 0) *bump_seq = *bump_seq + 1u;
  if (host_mirror != nullptr) {
    // result read-back without a copy-engine launch or a stream sync: the committed ledger page
    // goes to a pinned host page with plain PCIe posted writes, then a release-store of the new
    // epoch into the word the host is spinning on (engine/fused.py::run_round_e2e)
    constexpr int kWords = static_cast<int>(sizeof(RoundState) / 4);
    const volatile uint32_t* src = reinterpret_cast<const volatile uint32_t*>(st);
    for (int i = threadIdx.x; i < kWords; i += blockDim.x)
      asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(host_mirror + i), "r"(src[i]) : "memory");
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) ptx::st_release_sys(host_mirror + kMirrorSeqWord, epoch + 1);
  }
  // tell every peer that this rank no longer reads epoch `epoch` buffers
  if (threadIdx.x < n)
    ptx::st_release_sys(
        at<uint32_t>(f.peers.base[threadIdx.x], f.lay.flags_off) + FLAG_DONE + f.rank, epoch + 1);
  if (threadIdx.x == 0) stamp(plan, STAMP_CONS_END);
}

template <bool kRobust, int kServerOpt>
__global__ void __launch_bounds__(kFedThreads)
k_consensus(FedArgs f, int n_val, int weight_by_score, int two_shot, int use_mc,
            uint32_t* host_mirror, uint32_t* bump_seq, uint32_t agg, ServerOptArgs so) {
  consensus_body<kRobust, kServerOpt, DP_OFF>(f, n_val, weight_by_score, two_shot, use_mc, host_mirror, bump_seq,
                                               agg, so, DpArgs{}, nullptr);
}

template <bool kRobust, int kServerOpt, int kDp>
__global__ void __launch_bounds__(kFedThreads)
k_consensus_dp(FedArgs f, int n_val, int weight_by_score, int two_shot, int use_mc,
               uint32_t* host_mirror, uint32_t* bump_seq, uint32_t agg, ServerOptArgs so, DpArgs dp) {
  __shared__ DpShared dsh;
  consensus_body<kRobust, kServerOpt, kDp>(f, n_val, weight_by_score, two_shot, use_mc, host_mirror, bump_seq,
                                           agg, so, dp, &dsh);
}

// DP norms (launched right before k_consensus_dp): this rank's slice [lo, hi) of every admitted
// upload, d = u - g in fp32, d * d summed in fp64 per thread, per block in a fixed shuffle order, and
// the blocks' partials in block-index order by the last block, which pushes the result into every
// replica's DpPage and releases FLAG_NORM there.
__global__ void __launch_bounds__(kFedThreads) k_update_norms(FedArgs f, long long dp_off) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  char* me = f.peers.base[f.rank];
  const RoundState* st = at<RoundState>(me, f.lay.state_off);
  const RoundPlan* plan = at<RoundPlan>(me, f.lay.plan_off);
  const uint32_t* flags = at<uint32_t>(me, f.lay.flags_off);
  DpPage* page = at<DpPage>(me, dp_off);
  const uint32_t epoch = st->epoch;
  const uint32_t par = epoch & 1u;
  const int n = f.n_ranks;
  // the candidates exactly as k_consensus resolves them; the acquire makes each upload readable
  __shared__ int cand_of[kMaxRanks];
  __shared__ int n_cand;
  __shared__ bool last;
  __shared__ double warp_part[kFedThreads / 32][kMaxRanks];
  if (threadIdx.x == 0) {
    const bool fk = admit::first_k(st);
    const int nc = plan->n_cand;
    for (int z = 0; z < nc; ++z) {
      const int t = fk ? admit::wait_slot(admit::page(me, f.lay, par), z, epoch) : plan->cand_rank[z];
      ptx::wait_flag_ge(flags + FLAG_TRAINED + t, epoch + 1);
      cand_of[z] = t;
    }
    n_cand = nc;
  }
  __syncthreads();
  const int nc = n_cand;
  const float4* src[kMaxRanks];
#pragma unroll
  for (int z = 0; z < kMaxRanks; ++z)
    src[z] = at<const float4>(f.peers.base[z < nc ? cand_of[z] : f.rank], f.lay.upload_master_off[par]);
  const float4* g = at<const float4>(me, f.lay.global_off);
  const long long nv = f.lay.n_params / 4;
  const long long per = (nv + n - 1) / n;
  const long long lo = per * f.rank < nv ? per * f.rank : nv;
  const long long hi = lo + per < nv ? lo + per : nv;
  double acc[kMaxRanks];
#pragma unroll
  for (int z = 0; z < kMaxRanks; ++z) acc[z] = 0.0;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = lo + blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < hi; i += stride) {
    const float4 gv = g[i];
    float4 u[kMaxRanks];
#pragma unroll
    for (int z = 0; z < kMaxRanks; ++z)
      if (z < nc) u[z] = ptx::ld_peer_f4(src[z] + i);
#pragma unroll
    for (int z = 0; z < kMaxRanks; ++z)
      if (z < nc) {
        const double dx = so_sub(u[z].x, gv.x), dy = so_sub(u[z].y, gv.y);
        const double dz = so_sub(u[z].z, gv.z), dw = so_sub(u[z].w, gv.w);
        acc[z] += dx * dx;   // each square is exact in fp64
        acc[z] += dy * dy;
        acc[z] += dz * dz;
        acc[z] += dw * dw;
      }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int z = 0; z < kMaxRanks; ++z) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) acc[z] += __shfl_xor_sync(0xffffffffu, acc[z], o);
    if (lane == 0) warp_part[warp][z] = acc[z];
  }
  __syncthreads();
  if (threadIdx.x < kMaxRanks) {
    double s = 0.0;
    for (int w = 0; w < kFedThreads / 32; ++w) s += warp_part[w][threadIdx.x];
    page->block[blockIdx.x][threadIdx.x] = s;
    __threadfence();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned done = atomicAdd(&page->ticket, 1u);
    last = (done == gridDim.x - 1);
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  if (threadIdx.x < nc) {
    const int z = threadIdx.x;
    const volatile double* blk = &page->block[0][0];
    double s = 0.0;
    for (unsigned b = 0; b < gridDim.x; ++b) s += blk[b * kMaxRanks + z];
    for (int r = 0; r < n; ++r)
      at<DpPage>(f.peers.base[r], dp_off)->partial[par][f.rank][cand_of[z]] = s;
  }
  __syncthreads();   // every partial store before the releases (release patterns are cumulative)
  if (threadIdx.x == 0) page->ticket = 0u;
  if (threadIdx.x < n) {
    __threadfence_system();
    ptx::st_release_sys(at<uint32_t>(f.peers.base[threadIdx.x], f.lay.flags_off) + FLAG_NORM + f.rank, epoch + 1);
  }
}

__global__ void k_p2p_read(const float4* __restrict__ src, float4* __restrict__ dst, long long n) {
  const long long tid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = tid; i + 3 * stride < n; i += 4 * stride) {
    const float4 a = ptx::ld_peer_f4(src + i);
    const float4 b = ptx::ld_peer_f4(src + i + stride);
    const float4 c = ptx::ld_peer_f4(src + i + 2 * stride);
    const float4 d = ptx::ld_peer_f4(src + i + 3 * stride);
    dst[i] = a; dst[i + stride] = b; dst[i + 2 * stride] = c; dst[i + 3 * stride] = d;
  }
}
__global__ void k_mc_store(float4* mc_dst, const float4* __restrict__ src, long long n) {
  const long long tid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = tid; i < n; i += stride) ptx::multimem_st_f4(mc_dst + i, src[i]);
}

// Generic (non-captured) engines: block the stream until every trainer of the current epoch has
// published its upload, so ordinary kernels launched afterwards may read the peers' buffers.
__global__ void k_wait_trained(FedArgs f) {
  char* me = f.peers.base[f.rank];
  const RoundState* st = at<RoundState>(me, f.lay.state_off);
  const uint32_t* flags = at<uint32_t>(me, f.lay.flags_off);
  const int r = threadIdx.x;
  if (r < f.n_ranks && (st->role[r] & ROLE_TRAINER))
    ptx::wait_flag_ge(flags + FLAG_TRAINED + r, st->epoch + 1);
}

// Committee-side gather ("QueryAllUpdates", C:299-311) without NCCL: block (x, z) waits for
// candidate z's trainer flag, then streams that trainer's uploaded bf16 weights (and optionally
// the fp32 master) out of the peer's HBM into a local staging slot with 16-byte P2P loads.
// Every candidate is pulled exactly once per committee rank and as soon as ITS trainer is
// done -- the validation GEMMs then read local memory instead of re-fetching each weight tile
// over NVLink once per M-tile.
__global__ void __launch_bounds__(256)
k_pull(FedArgs f, uint4* stage_shadow, float4* stage_master, const long long* ranges, int n_ranges) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  char* me = f.peers.base[f.rank];
  const RoundState* st = at<RoundState>(me, f.lay.state_off);
  RoundPlan* plan = at<RoundPlan>(me, f.lay.plan_off);
  if (!(st->role[f.rank] & ROLE_COMM)) return;
  const int z = blockIdx.y;
  if (z >= plan->n_cand) return;
  if (blockIdx.x == 0 && z == 0 && threadIdx.x == 0) stamp(plan, STAMP_PULL_BEGIN);
  const uint32_t epoch = st->epoch;
  const uint32_t par = epoch & 1u;
  __shared__ int t_sh;
  if (threadIdx.x == 0) {
    const int tt = admit::first_k(st) ? admit::wait_slot(admit::page(me, f.lay, par), z, epoch) : plan->cand_rank[z];
    ptx::wait_flag_ge(at<uint32_t>(me, f.lay.flags_off) + FLAG_TRAINED + tt, epoch + 1);
    t_sh = tt;
  }
  __syncthreads();
  const int t = t_sh;
  const long long tid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  {
    const long long nv = f.lay.n_params / 8;  // 8 bf16 per 16 bytes
    const uint4* src = at<const uint4>(f.peers.base[t], f.lay.upload_shadow_off[par]);
    uint4* dst = stage_shadow + static_cast<long long>(z) * nv;
    // four peer loads in flight per thread: with one, a single candidate (2 GPUs) moved 150 GB/s
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    long long i = tid;
    for (; i + 3 * stride < nv; i += 4 * stride) {
      const float4 a = ptx::ld_peer_f4(s4 + i), b = ptx::ld_peer_f4(s4 + i + stride);
      const float4 c = ptx::ld_peer_f4(s4 + i + 2 * stride), d = ptx::ld_peer_f4(s4 + i + 3 * stride);
      d4[i] = a; d4[i + stride] = b; d4[i + 2 * stride] = c; d4[i + 3 * stride] = d;
    }
    for (; i < nv; i += stride) d4[i] = ptx::ld_peer_f4(s4 + i);
  }
  if (stage_master != nullptr) {
    const long long nv = f.lay.n_params / 4;
    const float4* src = at<const float4>(f.peers.base[t], f.lay.upload_master_off[par]);
    float4* dst = stage_master + static_cast<long long>(z) * nv;
    if (ranges == nullptr) {
      for (long long i = tid; i < nv; i += stride) dst[i] = ptx::ld_peer_f4(src + i);
    } else {
      // only the fp32 ranges a forward pass reads (biases, norm parameters, running statistics):
      // ranges[r] = {first float4, float4 count}; every matrix is consumed from the bf16 copy
      for (int r = blockIdx.x; r < n_ranges; r += gridDim.x) {
        const long long o = ranges[2 * r], n4 = ranges[2 * r + 1];
        for (long long i = threadIdx.x; i < n4; i += blockDim.x) dst[o + i] = ptx::ld_peer_f4(src + o + i);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) stamp(plan, STAMP_PULL_END);
}

// fp8 MLP variant: a candidate is one Mx8MlpLayout blob (e4m3 weights + scale chunks + fp32
// biases, 227 KB for 784x256x62) at heap offset off[parity] of its trainer.  Each byte of it
// crosses NVLink once; the weights land dequantised (exact bf16) in the local bf16 slot the
// validation maps cover, the biases in the local blob slot (epi::mx8_unpack_unit).
__global__ void __launch_bounds__(256)
k_pull_blob(FedArgs f, long long off0, long long off1, Mx8Unpack un, uint8_t* stage_blob, long long blob_bytes,
            __nv_bfloat16* stage_dq, long long stage_stride) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  char* me = f.peers.base[f.rank];
  const RoundState* st = at<RoundState>(me, f.lay.state_off);
  RoundPlan* plan = at<RoundPlan>(me, f.lay.plan_off);
  if (!(st->role[f.rank] & ROLE_COMM)) return;
  const int z = blockIdx.y;
  if (z >= plan->n_cand) return;
  if (blockIdx.x == 0 && z == 0 && threadIdx.x == 0) stamp(plan, STAMP_PULL_BEGIN);
  const uint32_t epoch = st->epoch;
  __shared__ int t_sh;
  if (threadIdx.x == 0) {
    const int tt = admit::first_k(st) ? admit::wait_slot(admit::page(me, f.lay, epoch & 1u), z, epoch)
                                      : plan->cand_rank[z];
    ptx::wait_flag_ge(at<uint32_t>(me, f.lay.flags_off) + FLAG_TRAINED + tt, epoch + 1);
    t_sh = tt;
  }
  __syncthreads();
  const int t = t_sh;
  const uint8_t* src = at<const uint8_t>(f.peers.base[t], (epoch & 1u) ? off1 : off0);
  uint8_t* dblob = stage_blob + static_cast<long long>(z) * blob_bytes;
  __nv_bfloat16* ddq = stage_dq + static_cast<long long>(z) * stage_stride;
  const long long n = epi::mx8_unpack_units(un);
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += stride)
    epi::mx8_unpack_unit(un, src, ddq, dblob, i);
  __syncthreads();
  if (threadIdx.x == 0) stamp(plan, STAMP_PULL_END);
}

int fed_grid(long long n_params) {
  // one 16-byte element per thread while the grid fits in ~4 resident blocks per SM: the copies
  // are latency-bound (small models), so every load should be in flight at once
  long long blocks = (n_params / 4 + kFedThreads * 2 - 1) / (kFedThreads * 2);
  if (blocks > 132 * 4) blocks = 132 * 4;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

}  // namespace

cudaError_t fed_plan_round(const FedArgs& f, const PlanLayer* layers, int n_layers,
                           int steps_per_round, int staged, cudaStream_t s, const PlanBlobs* blobs,
                           const float* stage_master) {
  if (n_layers > kMaxPlanLayers) return cudaErrorInvalidValue;
  PlanLayers pl{};
  pl.n = n_layers;
  pl.steps_per_round = steps_per_round;
  pl.staged = staged;
  pl.stage_master = stage_master;
  if (blobs != nullptr) {
    pl.use_blob = 1;
    pl.stage_blob = blobs->stage; pl.blob_bytes = blobs->bytes;
    pl.upq_off[0] = blobs->upq_off[0]; pl.upq_off[1] = blobs->upq_off[1];
  }
  for (int i = 0; i < n_layers; ++i) pl.l[i] = layers[i];
  note_launch();
  return launch_pdl(k_plan, dim3(1), dim3(32), 0, s, f, pl);
}

cudaError_t fed_upload(const FedArgs& f, int n_samples, int n_loss_terms, int byz_mode,
                       float byz_scale, cudaStream_t s, int straggle_us) {
  note_launch();
  return launch_pdl(k_upload, dim3(fed_grid(f.lay.n_params)), dim3(kFedThreads), 0, s, f, n_samples,
                    n_loss_terms, byz_mode, byz_scale, straggle_us);
}

template <bool kRobust>
static cudaError_t launch_consensus(int opt, dim3 grid, dim3 block, cudaStream_t s, const FedArgs& f, int n_val,
                                    int weight_by_score, int two_shot, int use_multicast, uint32_t* host_mirror,
                                    uint32_t* bump_seq, uint32_t agg, const ServerOptArgs& so) {
  switch (opt) {
    case SOPT_MOMENTUM:
      return launch_pdl(k_consensus<kRobust, SOPT_MOMENTUM>, grid, block, 0, s, f, n_val, weight_by_score, two_shot,
                        use_multicast, host_mirror, bump_seq, agg, so);
    case SOPT_ADAM:
      return launch_pdl(k_consensus<kRobust, SOPT_ADAM>, grid, block, 0, s, f, n_val, weight_by_score, two_shot,
                        use_multicast, host_mirror, bump_seq, agg, so);
    case SOPT_YOGI:
      return launch_pdl(k_consensus<kRobust, SOPT_YOGI>, grid, block, 0, s, f, n_val, weight_by_score, two_shot,
                        use_multicast, host_mirror, bump_seq, agg, so);
    default:
      return launch_pdl(k_consensus<kRobust, SOPT_NONE>, grid, block, 0, s, f, n_val, weight_by_score, two_shot,
                        use_multicast, host_mirror, bump_seq, agg, so);
  }
}

template <bool kRobust, int kDp>
static cudaError_t launch_consensus_dp(int opt, dim3 grid, dim3 block, cudaStream_t s, const FedArgs& f, int n_val,
                                       int weight_by_score, int two_shot, int use_multicast, uint32_t* host_mirror,
                                       uint32_t* bump_seq, uint32_t agg, const ServerOptArgs& so, const DpArgs& dp) {
  switch (opt) {
    case SOPT_MOMENTUM:
      return launch_pdl(k_consensus_dp<kRobust, SOPT_MOMENTUM, kDp>, grid, block, 0, s, f, n_val, weight_by_score,
                        two_shot, use_multicast, host_mirror, bump_seq, agg, so, dp);
    case SOPT_ADAM:
      return launch_pdl(k_consensus_dp<kRobust, SOPT_ADAM, kDp>, grid, block, 0, s, f, n_val, weight_by_score,
                        two_shot, use_multicast, host_mirror, bump_seq, agg, so, dp);
    case SOPT_YOGI:
      return launch_pdl(k_consensus_dp<kRobust, SOPT_YOGI, kDp>, grid, block, 0, s, f, n_val, weight_by_score,
                        two_shot, use_multicast, host_mirror, bump_seq, agg, so, dp);
    default:
      return launch_pdl(k_consensus_dp<kRobust, SOPT_NONE, kDp>, grid, block, 0, s, f, n_val, weight_by_score,
                        two_shot, use_multicast, host_mirror, bump_seq, agg, so, dp);
  }
}

// a DpPage offset every rank can use: positive, 16-byte aligned
static bool dp_off_ok(long long off) { return off > 0 && off % 16 == 0; }

cudaError_t fed_update_norms(const FedArgs& f, long long dp_off, cudaStream_t s) {
  if (!dp_off_ok(dp_off) || f.n_ranks < 1) return cudaErrorInvalidValue;
  note_launch();
  return launch_pdl(k_update_norms, dim3(fed_grid(f.lay.n_params / f.n_ranks)), dim3(kFedThreads), 0, s, f, dp_off);
}

cudaError_t fed_consensus_aggregate(const FedArgs& f, int n_val, int weight_by_score,
                                    int two_shot, int use_multicast, cudaStream_t s,
                                    uint32_t* host_mirror, uint32_t* bump_seq, int rule, int trim,
                                    const ServerOptArgs* so, const DpArgs* dp) {
  // robust rules are unweighted: a score weight would be silently ignored
  if (!agg_rule_valid(rule, trim) || (rule != AGG_FEDAVG && weight_by_score)) return cudaErrorInvalidValue;
  ServerOptArgs sa{};
  if (so != nullptr) sa = *so;
  if (*server_opt_check(sa.opt, sa.lr, sa.b1, sa.b2, sa.tau) != '\0') return cudaErrorInvalidValue;
  if (sa.opt != SOPT_NONE) {  // the state vectors: float4-aligned, v present for adam / yogi
    const bool need_v = server_state_vectors(sa.opt) == 2;
    if (sa.m_off <= 0 || sa.m_off % 16 != 0 || (need_v && (sa.v_off <= 0 || sa.v_off % 16 != 0)))
      return cudaErrorInvalidValue;
  }
  DpArgs da{};
  if (dp != nullptr) da = *dp;
  if (*dp_check(da.mode, da.clip, da.noise, rule) != '\0' || (da.mode != DP_OFF && !dp_off_ok(da.off)))
    return cudaErrorInvalidValue;
  const long long work = two_shot ? f.lay.n_params / (f.n_ranks > 0 ? f.n_ranks : 1)
                                  : f.lay.n_params;
  note_launch();
  const dim3 grid(fed_grid(work)), block(kFedThreads);
  const uint32_t agg = agg_word(rule, trim, sa.opt, da.mode);
  if (da.mode == DP_CLIP && rule == AGG_FEDAVG)
    return launch_consensus_dp<false, DP_CLIP>(sa.opt, grid, block, s, f, n_val, weight_by_score, two_shot,
                                               use_multicast, host_mirror, bump_seq, agg, sa, da);
  if (da.mode == DP_CLIP)
    return launch_consensus_dp<true, DP_CLIP>(sa.opt, grid, block, s, f, n_val, weight_by_score, two_shot,
                                              use_multicast, host_mirror, bump_seq, agg, sa, da);
  if (da.mode == DP_NOISE)   // FedAvg only (dp_check)
    return launch_consensus_dp<false, DP_NOISE>(sa.opt, grid, block, s, f, n_val, weight_by_score, two_shot,
                                                use_multicast, host_mirror, bump_seq, agg, sa, da);
  if (rule == AGG_FEDAVG)
    return launch_consensus<false>(sa.opt, grid, block, s, f, n_val, weight_by_score, two_shot, use_multicast,
                                   host_mirror, bump_seq, agg, sa);
  return launch_consensus<true>(sa.opt, grid, block, s, f, n_val, weight_by_score, two_shot, use_multicast,
                                host_mirror, bump_seq, agg, sa);
}

cudaError_t fed_pull_candidates(const FedArgs& f, void* stage_shadow, float* stage_master,
                                cudaStream_t s, const long long* ranges, int n_ranges) {
  long long blocks = (f.lay.n_params / 8 + 256 * 4 - 1) / (256 * 4);
  if (blocks > 74) blocks = 74;  // x kMaxRanks candidates in flight
  if (blocks < 1) blocks = 1;
  note_launch();
  return launch_pdl(k_pull, dim3(static_cast<unsigned>(blocks), kMaxRanks), dim3(256), 0, s, f,
                    reinterpret_cast<uint4*>(stage_shadow),
                    reinterpret_cast<float4*>(stage_master), ranges, n_ranges);
}

cudaError_t fed_pull_blobs(const FedArgs& f, long long off0, long long off1, const Mx8Unpack& un,
                           void* stage_blob, long long blob_bytes, void* stage_dq, long long stage_stride,
                           cudaStream_t s) {
  if (un.in_dim % 16 != 0 || un.hidden % 32 != 0 || un.b1 + 4LL * un.hidden + 256 > blob_bytes) return cudaErrorInvalidValue;
  long long blocks = (epi::mx8_unpack_units(un) + 256 * 2 - 1) / (256 * 2);
  if (blocks > 18) blocks = 18;  // x kMaxRanks candidate slots <= 144 blocks: one wave
  if (blocks < 1) blocks = 1;
  note_launch();
  return launch_pdl(k_pull_blob, dim3(static_cast<unsigned>(blocks), kMaxRanks), dim3(256), 0, s, f, off0, off1, un,
                    static_cast<uint8_t*>(stage_blob), blob_bytes, static_cast<__nv_bfloat16*>(stage_dq),
                    stage_stride);
}

cudaError_t fed_wait_trained(const FedArgs& f, cudaStream_t s) {
  (void)cudaGetLastError();
  k_wait_trained<<<1, 32, 0, s>>>(f);
  note_launch();
  return cudaGetLastError();
}

cudaError_t p2p_read_probe(const float4* peer_src, float4* local_dst, int64_t n_vec,
                           cudaStream_t s) {
  k_p2p_read<<<132 * 4, 256, 0, s>>>(peer_src, local_dst, n_vec);
  note_launch();
  return cudaGetLastError();
}
cudaError_t mc_store_probe(float4* mc_dst, const float4* local_src, int64_t n_vec,
                           cudaStream_t s) {
  k_mc_store<<<132 * 4, 256, 0, s>>>(mc_dst, local_src, n_vec);
  note_launch();
  return cudaGetLastError();
}

}  // namespace bflc
