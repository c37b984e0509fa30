// One persistent kernel for a trainer's whole local-training pass of the 2-layer MLP:
// every mini-batch step (forward, softmax-xent, both weight gradients, the hidden gradient
// and the optimizer) runs inside ONE launch; phases are separated by a device-wide barrier
// instead of kernel boundaries -- and the LAST step's optimizer epilogue is also the
// UploadLocalUpdate of the protocol (reference: CommitteePrecompiled.cpp:215-258): it writes the
// peer-readable upload buffers and CTA 0 releases FLAG_TRAINED on every peer.
//
//   per step:  P1  h  = relu(x W1^T + b1)                       K = 784
//              X   per M-tile of batch rows, 4 CTAs: fwd2 -> softmax-xent -> dh = (dlogits W2) relu'(h)
//              B   dW1 = dh^T x  ||  dW2 = dlogits^T h  as 64 x 64 tiles (one m64 wgmma) on 57 CTAs,
//                  optimizer (SGD / Adam) applied to the fp32 master straight from the
//                  accumulator tile (E_OPT) + compute-copy refresh
//
// Plan 4 (the default) launches 4-CTA clusters and runs P1 and X of a 64-row M-tile in one cluster:
// the four P1 CTAs of an M-tile ARE its four chain CTAs, so each writes its 64 x 64 slice of h into
// its own h tile and bulk-copies it (TMA engine, distributed shared memory) into the h tiles of the
// other three, instead of storing it to global memory, crossing a grid barrier and TMA-loading the
// 32 KB tile back.  Two mbarriers order the hand-over: ring_free (every MMA warp of the cluster has
// retired its last fwd1 wgmma, so no ring stage of any CTA is still read) before the copies, and hx
// (own slice written + the three peers' 24 KB landed) before fwd2.  Per-thread DSMEM stores were
// measured slower than the grid barrier they replace; so was a cluster-scope release per arrive,
// which costs a GPU-scope memory barrier.  64-row M-tiles (plans 0 and 3: 128) put fwd1 and the
// chain on twice the CTAs, and their epilogues' serial per-row work on twice the threads per row.
//
// Precision.  bf16 mode: every GEMM is a bf16 wgmma on bf16 shadows.  fp8 mode (BASELINE.json
// config #2, "block-scaled fp8", MXFP8): fwd1 and fwd2 multiply MXFP8-quantised operands, but
// Hopper has no block-scaled MMA, so they run the same bf16 wgmma mainloop on exactly
// dequantised copies: bf16(e4m3 * 2^(s-127)) is exact for every scale byte the quantisers emit
// (epi::mx8_dq4), and an fp32-accumulating bf16 wgmma over those copies forms the block-scaled
// product.  x_dq comes from the input kernel (elementwise_optim.cu); the E_OPT epilogue
// re-quantises every updated weight tile (two lanes per 32-element K-group of the staged tile:
// amax, one scale byte, 32 e4m3 bytes into the MXFP8 blob) and stores the dequantised values into
// work_dq; the fwd1 epilogue quantises h and stores h_dq.  The hidden/weight gradients stay bf16,
// masters and Adam moments fp32.  FP8 (the template flag) selects only these epilogues.
//
// Warp roles (512 threads, four warpgroups): warps 0-3 = the MMA warpgroup (accumulators in
// registers, parked in a shared-memory accumulator tile, wgmma.cuh AccTile, once a tile's
// reduction is done; setmaxnreg.inc); warps 4-11 = the two epilogue warpgroups; warps 12-15 = the
// producer warpgroup (setmaxnreg.dec), whose warp 12 issues the TMA.  Each role runs its own copy
// of the step loop, so no wgmma sits under a warp-dependent branch.  Epilogue warp (q, half) owns
// rows 32q .. 32q+31 of the tile and the column half `half` (columns [32h, 32h+32)).
//
// Each GEMM tile is the same wgmma / TMA pipeline as gemm_sm100.cu (5-stage 128B-swizzled ring,
// staged coalesced epilogue); the smem ring, its mbarriers and the accumulator tile persist
// across tiles, phases and steps.  Every CTA runs at most one tile per phase, so the accumulator
// tile is never written while an epilogue still reads it.
//
// Why: at this problem size every stand-alone GEMM launch costs several microseconds of which
// only a fraction is math (launch, prologue, first-TMA latency, drain) -- six launches per step.
// Inside one kernel the fixed costs are paid once and a phase boundary is a grid barrier.
// (Reference step: python-sdk/main.py:141-148, three sess.run calls; Adam: the commented
// alternative at python-sdk/main.py:126.)
#include <cuda_bf16.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "bflc_kernels.h"
#include "consensus_math.hpp"
#include "epi_common.cuh"
#include "fed_admit.cuh"
#include "launch.cuh"
#include "sm100_ptx.cuh"
#include "wgmma.cuh"

namespace bflc {

namespace {

using epi::kStgLd;
using epi::stage_put;
using epi::stage_get;
using epi::col_sum32;
using epi::st_sw128;
__device__ __forceinline__ uint32_t pack2(float a, float b) { return epi::pack_bf16x2(a, b); }

constexpr int kBM = 128, kBN = 64, kStages = 5;
constexpr int kABytes = kBM * 128, kBBytes = kBN * 128, kStageBytes = kABytes + kBBytes;
constexpr int kTileBytes = kStages * kStageBytes;
constexpr int kBarBytes = 512;
constexpr int kEpiWarps = 8;       // two per row quarter: warp (q, half) owns 32 of a tile's 64 columns
constexpr int kEpiThreads = kEpiWarps * 32;
constexpr int kStgAll = kEpiWarps * 32 * kStgLd * 4;
constexpr int kBiasFloats = 320;   // chain: b1[256] | b2[64]; tile jobs use the first kBN
constexpr int kAccPitch = kBN + 4;                  // fp32 accumulator tile [128][68]
constexpr int kAccBytes = kBM * kAccPitch * 4;
// chain column sums (db1, db2): the staging buffers re-cut as one fp32 [rows][kRedLd] tile
constexpr int kRedLd = kBN + 4;
static_assert(kBM * kRedLd * 4 <= kStgAll, "column-sum tile");
constexpr int kSmemTotal = kTileBytes + kBarBytes + kStgAll + kBiasFloats * 4 + kAccBytes + 1024;
static_assert(kSmemTotal <= 227 * 1024, "shared memory budget");
// FedProx launches only, behind the accumulator tile: a weight-gradient tile's anchor (128 x 64 fp32), or
// on a 64-row tile its anchor and master (prox_stage)
constexpr int kProxBytes = kBM * kBN * 4;
constexpr int kSmemProx = kSmemTotal + kProxBytes;
static_assert(kSmemProx <= 227 * 1024, "shared memory budget (FedProx)");
constexpr int kEpiT0 = 128;        // first epilogue thread (warpgroup 0 = the MMA warpgroup)
constexpr int kProducerWarp = 4 + kEpiWarps;   // first warp of the producer warpgroup: issues the TMA
constexpr int kThreads = kEpiT0 + kEpiThreads + 128;
// Registers per thread after setmaxnreg (the launch gives every thread 65536 / 512 = 128): the
// producer warpgroup hands its surplus to the MMA warpgroup, which holds two 128 x 64 fp32
// accumulators, and to the two epilogue warpgroups.
constexpr int kProducerRegs = 40, kMmaRegs = 184, kEpiRegs = 144;
static_assert(kProducerRegs + kMmaRegs + 2 * kEpiRegs <= 4 * 128, "register file");
enum Role : int { kRoleProducer = 0, kRoleMma = 1, kRoleEpi = 2 };
constexpr int kGrid = 32;

// ---- fused chain (hidden == 256): the ring memory re-cut as
//   [0, 64 KB) h tile = fwd2's A operand | [64, 96 KB) W2 K-major (fwd2's B) | [96, 104 KB) this
//   CTA's 64-column slice of W2 MN-major (dh's B) | [104, 120 KB) dlogits (dh's A).
// Sized for plan 3's 128-row M-tiles; plan 4's 64-row tiles use the first half of the h and dlogits
// regions (K-block kb of h at kOffH + kb * 8 KB), so both plans share one map.
constexpr int kOffH = 0;
constexpr int kOffW2K = 64 * 1024;
constexpr int kOffW2MN = 96 * 1024;
constexpr int kOffDL = 104 * 1024;
static_assert(kOffDL + 16384 <= kTileBytes, "chain smem layout");
constexpr int kChainH = 256;
constexpr int kDefaultPlan = 4;    // phase plan when neither the caller nor BFLC_MLP_CHAIN picks one (0 | 3 | 4)
constexpr int kCluster = 4;        // plan 4: CTAs per cluster = the chain CTAs of one M-tile
constexpr int kBMx = 64;           // plan 4: M-tile height of fwd1 and the chain
constexpr int kHSlice = kBMx * 128;   // plan 4: one CTA's 64-column slice of the h tile (bf16, swizzled)

enum EpiMode : int { E_BIAS_RELU_BF16 = 0, E_XENT = 1, E_F32 = 2, E_MASK_COLSUM_BF16 = 3,
                     E_OPT = 4 };  // E_OPT: the tile IS the gradient -> optimizer applied in the epilogue

struct Maps {  // TMA descriptors, SWIZZLE_128B, all bf16.  fp8 mode: x_k, w1_k, h_k and w2_k cover
               // the dequantised copies x_dq, work_dq and h_dq
  CUtensorMap x_k, w1_k, h_k, w2_k, dl_mn, h_mn, dl_k, w2_mn, dh_mn, x_mn;
};

struct Args {
  int B, steps, in_dim, hidden, n_classes, ncp;  // ncp = dlogits row stride (padded classes)
  int epoch_steps;               // E: step s reads rows [(s mod E) B, (s mod E) B + B) of x and the labels
  int chain;                     // 0: P1|P2|P3 as separate phases   3: P1 | fwd2->xent->dh chained
                                 // 4: as 3, P1 and the chain in one cluster, h handed over on chip
  int epiopt;                    // optimizer applied in the weight-gradient epilogues (no P5)
  unsigned long long* dbg;       // optional %globaltimer stamps [steps][32] written by CTA 0
  const unsigned int* x_ready;   // optional input pipeline: step s may read x once x_ready[s mod E] >= *round_seq + 1
  const unsigned int* round_seq;
  long long n_params;
  const int* pred;               // whole kernel is a no-op when *pred == 0 (non-trainer rank)
  unsigned int* barrier;         // device-wide phase barrier counter (zeroed before launch)
  // parameters / optimizer state
  float* master; const float* b1; const float* b2;
  float* grad; float* gw1; float* gb1; float* gw2; float* gb2;
  __nv_bfloat16* shadow;
  float* adam_m; float* adam_v;
  int adam; float lr, beta1, beta2, eps; const int* step_base;
  // activations
  __nv_bfloat16* h; __nv_bfloat16* dlogits; __nv_bfloat16* dh;
  const int32_t* labels;
  float* loss_sum; unsigned int* correct;
  // fp8 forward: the MXFP8 blob of the weights, their dequantised copy (W1 [hidden][in_dim], then
  // W2 [64][hidden]) and the dequantised e4m3 h of the current step
  uint8_t* work_q; __nv_bfloat16* work_dq; __nv_bfloat16* h_dq;
  Mx8MlpLayout ql;
  int bm_w;                      // weight-gradient tile height: 64 (default) or 128
  // fused upload
  int has_fed; FedArgs f; long long upq_off[2];
  int n_samples, n_loss_terms, byz_mode; float byz_scale; int straggle_us;
  const float* prox_anchor; float prox_mu;   // FedProx (MlpRoundArgs); null: no proximal term
};

// DP-SGD (mlp_dpsgd_round_kernel only; plan 4 with the optimizer in the epilogue, hidden == 256).  Per
// example n of a step, from its bf16 rows as stored before clipping (x_n, h_n, dlogits dz_n, masked dh_n):
//   site 0 (fc2):  a = ||dz_n||^2, b = ||h_n||^2 + 1   site 1 (fc1):  a = ||dh_n||^2, b = ||x_n||^2 + 1
//   sq = a b, ab = sqrt(a) sqrt(b);  c_n = dpsgd_clip_factor(sq0 + sq1, ab0 + ab1, B, clip)
// as the generic MLP records its two R = 1 sites (k_pe_rows, k_dpsgd_clip).  dz' = bf16(dz c), dh' = bf16(dh c)
// (exact +0 where c = 0, whose h row is zeroed too); the bias gradients are fixed-order sums of 32-row
// column sums in bias_ws; the weight-gradient epilogues and the bias CTA add sigma xi_i, xi_i =
// dp_gauss4(seed, step word, i / 4, kDpsgdSite)[i % 4], before any proximal term.
struct TrainerDp {
  float clip, sigma, bsz;        // C, z C / B (0: no noise), B
  unsigned long long seed;       // the client's secret noise key
  const __nv_bfloat16* x;        // bf16 x [epoch rows][in_dim] (||x_n||^2; fp8 mode too)
  int* dropped;                  // examples with a non-finite bound
  float* bias_ws;                // [2 * M-tiles][hidden + 64]: 32-row column sums of dh' | dz'
  float* dbg;                    // optional: [steps][5][B] sq0, sq1, ab0, ab1, c, then the last step's
                                 // released gradient [n_params] (noise added, before any proximal term)
};
constexpr int kDpWsLd = kChainH + 64;
// plan 4's unused second half of the dlogits region: the per-row partials (||h||^2, ||x||^2, ||dh||^2) of
// the four slices [4][64] float4, this CTA's own fwd1 partials [64][2], and c [64]
constexpr int kOffDpX = kOffDL + 8192;
constexpr int kOffDpOwn = kOffDpX + 4 * 64 * 16;
constexpr int kOffDpC = kOffDpOwn + 64 * 8;
static_assert(kOffDpC + 64 * 4 <= kTileBytes, "DP-SGD exchange layout");

struct Job {  // one output tile (bm rows x 64 columns)
  const CUtensorMap* ta; const CUtensorMap* tb;
  int a_mn, b_mn;
  int a_c0, a_c1, b_c0, b_c1;   // TMA coordinates of K-block 0 (c0 = innermost)
  int n_kb;
  int m0, n0, M, N;             // output tile origin / logical extent
  int bm;                       // tile height: 128, or 64 (one m64 wgmma)
  int mode;
  long long ldd;
  void* d;                      // output
  const float* bias;            // E_BIAS_RELU_BF16 / E_XENT
  const __nv_bfloat16* aux;     // E_MASK_COLSUM_BF16: relu mask source, same shape as d
  float* colsum;
  const int32_t* labels;        // E_XENT (already offset to this step's rows)
  float grad_scale;
  float bc1, bc2;               // E_OPT + Adam: bias corrections of this step
  // ---- E_OPT in fp8 mode: where the re-quantised tile goes (byte offsets inside a model blob,
  // element offset of the matrix inside work_dq)
  int q_off, qsf_off, ldq, q_nkb;
  long long dq_off;
  int last;                     // last step of the round: E_OPT also publishes the upload
  int shadow;                   // E_OPT: refresh the bf16 shadow (see the W1 job in phase B)
  unsigned long long* dbg;      // this step's stamp slots (CTA 0): [dbg_slot] accumulator ready, [+1] epilogue done
  int dbg_slot;
};

struct Pipe {  // persistent pipeline state of one role
  uint32_t it;    // K-blocks processed so far (ring slot / parity)
  uint32_t tile;  // tiles processed so far (accumulator barrier parity)
};
struct ChainBars {
  uint64_t* h;                       // h tile (+ scale chunks) landed
  uint64_t* w2k; uint64_t* w2mn;     // W2 operand tiles landed
  uint64_t* acc_l; uint64_t* dl_ready; uint64_t* acc_dh;
  // plan 4: ring_free collects one arrive per MMA warp of every CTA of the cluster (4 x 4); hx one
  // arrive.expect_tx by a local epilogue thread plus the peers' bulk-copy bytes (3 x 8 KB)
  uint64_t* ring_free; uint64_t* hx;
};

template <typename T>
__device__ __forceinline__ T* heap_at(char* base, long long off) {
  return reinterpret_cast<T*>(base + off);
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Where the last step's optimizer epilogue publishes (resolved from the ledger page: the upload
// buffers are double-buffered by epoch parity).
struct UploadDst {
  float* master;            // fp32 upload (FedAvg operand)
  __nv_bfloat16* shadow;    // bf16 upload: the validation operand (fp8 mode: the blob dequantised)
  uint8_t* blob;            // fp8 mode: Mx8MlpLayout blob (what a staged committee pulls)
  const float* global;      // Byzantine fault injection: upload global - s * (w - global)
  float byz_scale;
};
template <bool FP8>
__device__ __forceinline__ UploadDst upload_dst(const Args& a) {
  char* me = a.f.peers.base[a.f.rank];
  const RoundState* st = heap_at<const RoundState>(me, a.f.lay.state_off);
  const uint32_t par = st->epoch & 1u;
  UploadDst u;
  u.master = heap_at<float>(me, a.f.lay.upload_master_off[par]);
  u.shadow = heap_at<__nv_bfloat16>(me, a.f.lay.upload_shadow_off[par]);
  u.blob = FP8 ? heap_at<uint8_t>(me, a.upq_off[par]) : nullptr;
  u.global = a.byz_mode == 1 ? heap_at<const float>(me, a.f.lay.global_off) : nullptr;
  u.byz_scale = a.byz_scale;
  return u;
}

// ---------------------------------------------------------------- producer / MMA / epilogue
__device__ __forceinline__ void produce_tile(const Job& j, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                             Pipe& pp) {
  const uint32_t a_bytes = static_cast<uint32_t>(j.bm) * 128u;
  for (int i = 0; i < j.n_kb; ++i, ++pp.it) {
    const int s = pp.it % kStages;
    const uint32_t ph = (pp.it / kStages) & 1;
    ptx::mbar_wait(&empty_bar[s], ph ^ 1);
    uint8_t* sa = smem + s * kStageBytes;
    uint8_t* sb = sa + kABytes;
    if (ptx::elect_one()) {
      ptx::mbar_expect_tx(&full_bar[s], a_bytes + kBBytes);
      if (!j.a_mn) {
        // K-major A: one 64-row box per m64 half (the 128B swizzle repeats every 8 rows, so two
        // boxes 8 KB apart are the layout of one 128-row box)
        ptx::tma_load_3d(sa, j.ta, &full_bar[s], j.a_c0 + i * 64, j.a_c1, 0);
        if (j.bm == kBM) ptx::tma_load_3d(sa + 64 * 128, j.ta, &full_bar[s], j.a_c0 + i * 64, j.a_c1 + 64, 0);
      } else {
        // MN-major A: one 64-element (128-byte) chunk of M per box
        ptx::tma_load_3d(sa, j.ta, &full_bar[s], j.a_c0, j.a_c1 + i * 64, 0);
        if (j.bm == kBM) ptx::tma_load_3d(sa + 64 * 128, j.ta, &full_bar[s], j.a_c0 + 64, j.a_c1 + i * 64, 0);
      }
      if (!j.b_mn)
        ptx::tma_load_3d(sb, j.tb, &full_bar[s], j.b_c0 + i * 64, j.b_c1, 0);
      else
        ptx::tma_load_3d(sb, j.tb, &full_bar[s], j.b_c0, j.b_c1 + i * 64, 0);
    }
    __syncwarp();
  }
}

// m64 accumulator rows -> accumulator-tile lanes: bm = 128 -> rows 64h + r; bm = 64 -> row m in
// lane (m % 16) + 32 (m / 16), i.e. the first 16 lanes of each row quarter
__device__ __forceinline__ int lane128(int r) { return r; }
__device__ __forceinline__ int lane128_hi(int r) { return 64 + r; }
__device__ __forceinline__ int lane64(int r) { return (r & 15) + 32 * (r >> 4); }

// FedProx: the gradient the optimizer consumes, g' = fma(mu, w - w0, g) (w the master before the step,
// w0 the anchor).  Every site tests prox_anchor first, so without one g is used as it is.
__device__ __forceinline__ float prox_grad(float g, float w, float w0, float mu) {
  return __fmaf_rn(mu, __fsub_rn(w, w0), g);
}
// 16-byte global -> shared copy that bypasses L1 and the registers; !ok writes zeros and reads nothing
__device__ __forceinline__ void cp_async16(uint32_t dst, const float* src, bool ok) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr)
               : "memory");
  return v;
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// FedProx on a weight-gradient tile (E_OPT), applied by the MMA warpgroup, which has registers to
// spare and nothing to do between its last wgmma and the epilogue's update: at the start of the tile
// its 128 threads cp.async the tile's anchor -- and on a 64-row tile the master too -- into the
// shared-memory region behind the accumulator tile (present only in FedProx launches); once the
// accumulators are in the tile they rewrite every gradient g there as g' = fma(mu, w - w0, g), then
// release the tile to the epilogue, whose update runs as without the term.  (The term inside the
// epilogue's update loop grew its spills past the ceilings of test_trainer_ptxas.py, however the
// anchor was fetched.)  Element e (float4) of the tile: row e / 16, columns 4 (e % 16) .. + 3.
__device__ __forceinline__ uint32_t prox_region(const wg::AccTile& at) { return ptx::smem_u32(at.p + kBM * kAccPitch); }

__device__ __forceinline__ void prox_stage(const Job& j, const Args& a, const wg::AccTile& at) {
  const long long pbase = reinterpret_cast<const float*>(j.d) - a.master;
  const uint32_t base = prox_region(at);
  const bool master = j.bm == 64;                 // anchor and master: 2 x 16 KB of the 32 KB region
  for (int e = threadIdx.x; e < j.bm * (kBN / 4); e += 128) {
    const int rw = j.m0 + (e >> 4), col = j.n0 + (e & 15) * 4;
    const bool ok = rw < j.M && col + 3 < j.N;
    const long long pi = pbase + static_cast<long long>(rw) * j.ldd + col;
    cp_async16(base + 16u * e, ok ? a.prox_anchor + pi : a.prox_anchor, ok);
    if (master) cp_async16(base + 16u * (e + kBM * kBN / 8), ok ? a.master + pi : a.master, ok);
  }
  cp_async_commit();
}

__device__ __forceinline__ void prox_apply(const Job& j, const Args& a, const wg::AccTile& at) {
  cp_async_wait_all();                                  // this thread's slots
  asm volatile("bar.sync 2, 128;" ::: "memory");        // every MMA thread's accumulators are in the tile
  const long long pbase = reinterpret_cast<const float*>(j.d) - a.master;
  const uint32_t base = prox_region(at);
  const bool master = j.bm == 64;
  for (int e = threadIdx.x; e < j.bm * (kBN / 4); e += 128) {
    const int r = e >> 4, c = (e & 15) * 4;
    const int rw = j.m0 + r, col = j.n0 + c;
    if (rw >= j.M || col + 3 >= j.N) continue;
    const float4 w0 = lds128(base + 16u * e);
    const float4 w = master ? lds128(base + 16u * (e + kBM * kBN / 8))
                            : __ldcg(reinterpret_cast<const float4*>(a.master + pbase + static_cast<long long>(rw) * j.ldd + col));
    float4* gp = reinterpret_cast<float4*>(at.p + (j.bm == 64 ? lane64(r) : r) * at.pitch + c);
    float4 g = *gp;
    g.x = prox_grad(g.x, w.x, w0.x, a.prox_mu); g.y = prox_grad(g.y, w.y, w0.y, a.prox_mu);
    g.z = prox_grad(g.z, w.z, w0.z, a.prox_mu); g.w = prox_grad(g.w, w.w, w0.w, a.prox_mu);
    *gp = g;
  }
}

// DP-SGD on a weight-gradient tile (E_OPT), by the MMA warpgroup once its accumulators are in the tile:
// g += sigma xi_i over the tile's flat indices i (a thread's 4 columns are one dp_gauss4 call: the W1 / W2
// offsets and row pitches are multiples of 4), and on the last step the released gradient -> dbg_grad.
// Runs before prox_apply (same element partition), so the proximal term comes after the noise.
__device__ __forceinline__ void dp_tile(const Job& j, const Args& a, const TrainerDp& d, uint32_t word,
                                        float* dbg_grad, const wg::AccTile& at) {
  asm volatile("bar.sync 2, 128;" ::: "memory");        // every MMA thread's accumulators are in the tile
  const long long pbase = reinterpret_cast<const float*>(j.d) - a.master;
  for (int e = threadIdx.x; e < j.bm * (kBN / 4); e += 128) {
    const int r = e >> 4, c = (e & 15) * 4;
    const int rw = j.m0 + r, col = j.n0 + c;
    if (rw >= j.M || col + 3 >= j.N) continue;
    const long long pi = pbase + static_cast<long long>(rw) * j.ldd + col;
    float4* gp = reinterpret_cast<float4*>(at.p + (j.bm == 64 ? lane64(r) : r) * at.pitch + c);
    float4 g = *gp;
    if (d.sigma > 0.f) {
      float z[4];
      dp_gauss4(d.seed, word, static_cast<uint64_t>(pi >> 2), z, kDpsgdSite);
      g.x = so_add(g.x, so_mul(d.sigma, z[0])); g.y = so_add(g.y, so_mul(d.sigma, z[1]));
      g.z = so_add(g.z, so_mul(d.sigma, z[2])); g.w = so_add(g.w, so_mul(d.sigma, z[3]));
      *gp = g;
    }
    if (dbg_grad != nullptr) *reinterpret_cast<float4*>(dbg_grad + pi) = g;
  }
}

// MMA warpgroup: one bm x 64 tile, rows 0-63 / 64-127 as two m64 wgmma sharing the B descriptor.
// ring_free (plan 4's fwd1): once the last wgmma has retired, one lane per warp tells every CTA of
// the cluster that this CTA's ring is no longer read.
// DP: pdp (DP-SGD entry, phase-B tiles) adds the noise / takes the hook (dp_tile) first.
template <bool DP = false>
__device__ __forceinline__ void mma_tile(const Job& j, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                         uint64_t* accum_bar, const wg::AccTile& at, Pipe& pp,
                                         uint64_t* ring_free = nullptr, const Args* pa = nullptr,
                                         const TrainerDp* pdp = nullptr, uint32_t dp_word = 0,
                                         float* dp_grad = nullptr) {
  // FedProx: pa is the kernel's Args on weight-gradient tiles of a launch with an anchor
  const bool prox = pa != nullptr && j.mode == E_OPT && pa->prox_anchor != nullptr;
  if (prox) prox_stage(j, *pa, at);
  float acc0[32], acc1[32];
  wg::zero(acc0);
  wg::zero(acc1);
  const uint32_t base = ptx::smem_u32(smem);
  const bool two = j.bm == kBM;   // CTA-uniform
  auto stage = [&](uint32_t it) { return base + (it % kStages) * static_cast<uint32_t>(kStageBytes); };
  // one K-block of wgmma stays in flight: a stage is released once the next K-block's wait<1>
  // shows that its wgmma have retired
  const uint32_t lbo_a = j.a_mn ? 8192u : 16u, lbo_b = j.b_mn ? 8192u : 16u;
  const uint32_t ks_a = j.a_mn ? 2048u : 32u, ks_b = j.b_mn ? 2048u : 32u;
  for (int i = 0; i < j.n_kb; ++i, ++pp.it) {
    const int s = pp.it % kStages;
    const uint32_t ph = (pp.it / kStages) & 1;
    ptx::mbar_wait(&full_bar[s], ph);
    const uint32_t sa = stage(pp.it), sb = sa + kABytes;
    wg::fence();
#pragma unroll
    for (uint32_t k = 0; k < 4; ++k) {
      const uint64_t bd = wg::desc(sb + k * ks_b, lbo_b);
      const uint32_t acc = (i > 0 || k > 0) ? 1u : 0u;
      wg::mma_bf16_rt<64>(acc0, wg::desc(sa + k * ks_a, lbo_a), bd, acc, j.a_mn, j.b_mn);
      if (two) wg::mma_bf16_rt<64>(acc1, wg::desc(sa + 8192u + k * ks_a, lbo_a), bd, acc, j.a_mn, j.b_mn);
    }
    wg::commit();
    wg::wait<1>();
    if (i > 0) ptx::mbar_arrive(&empty_bar[(pp.it - 1) % kStages]);
  }
  wg::wait<0>();
  wg::reg_fence(acc0);
  wg::reg_fence(acc1);
  if (j.n_kb > 0) ptx::mbar_arrive(&empty_bar[(pp.it - 1) % kStages]);
  if (ring_free != nullptr) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0)
      for (uint32_t r = 0; r < kCluster; ++r) ptx::mbar_arrive_remote(ring_free, r);
  }
  if (two) {
    wg::acc_put<64>(at, 0, acc0, lane128);
    wg::acc_put<64>(at, 0, acc1, lane128_hi);
  } else {
    wg::acc_put<64>(at, 0, acc0, lane64);
  }
  if constexpr (DP) {
    if (pdp != nullptr && j.mode == E_OPT && (pdp->sigma > 0.f || dp_grad != nullptr))
      dp_tile(j, *pa, *pdp, dp_word, dp_grad, at);
  }
  if (prox) prox_apply(j, *pa, at);
  ptx::mbar_arrive(accum_bar);
  ++pp.tile;
}

// SGD / Adam on n (<= 4) consecutive parameters starting at flat index pi, gradient in g[]:
// fp32 master, bf16 shadow (and the Adam moments) are updated in place; the new values are
// returned in w[].  Coherent loads: other CTAs of this kernel wrote these buffers in earlier phases.
__device__ __forceinline__ void opt_apply(const Args& a, long long pi, int n, const float* g,
                                          float bc1, float bc2, float (&w)[4]) {
  float m[4], v[4];
  const bool vec = n == 4 && (pi & 3) == 0;
  if (vec) {
    const float4 w4 = __ldcg(reinterpret_cast<const float4*>(a.master + pi));
    w[0] = w4.x; w[1] = w4.y; w[2] = w4.z; w[3] = w4.w;
    if (a.adam) {
      const float4 m4 = __ldcg(reinterpret_cast<const float4*>(a.adam_m + pi));
      const float4 v4 = __ldcg(reinterpret_cast<const float4*>(a.adam_v + pi));
      m[0] = m4.x; m[1] = m4.y; m[2] = m4.z; m[3] = m4.w;
      v[0] = v4.x; v[1] = v4.y; v[2] = v4.z; v[3] = v4.w;
    }
  } else {
    for (int k = 0; k < n; ++k) {
      w[k] = __ldcg(a.master + pi + k);
      if (a.adam) { m[k] = __ldcg(a.adam_m + pi + k); v[k] = __ldcg(a.adam_v + pi + k); }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (k >= n) break;
    float gk = g[k];
    if (a.prox_anchor != nullptr) gk = prox_grad(gk, w[k], __ldcg(a.prox_anchor + pi + k), a.prox_mu);
    if (a.adam) {
      m[k] = a.beta1 * m[k] + (1.f - a.beta1) * gk;
      v[k] = a.beta2 * v[k] + (1.f - a.beta2) * gk * gk;
      w[k] -= a.lr * (m[k] / bc1) / (sqrtf(v[k] / bc2) + a.eps);
    } else {
      w[k] -= a.lr * gk;
    }
  }
  if (vec) {
    *reinterpret_cast<float4*>(a.master + pi) = make_float4(w[0], w[1], w[2], w[3]);
    *reinterpret_cast<uint2*>(a.shadow + pi) = make_uint2(pack2(w[0], w[1]), pack2(w[2], w[3]));
    if (a.adam) {
      *reinterpret_cast<float4*>(a.adam_m + pi) = make_float4(m[0], m[1], m[2], m[3]);
      *reinterpret_cast<float4*>(a.adam_v + pi) = make_float4(v[0], v[1], v[2], v[3]);
    }
  } else {
    for (int k = 0; k < n; ++k) {
      a.master[pi + k] = w[k];
      a.shadow[pi + k] = __float2bfloat16(w[k]);
      if (a.adam) { a.adam_m[pi + k] = m[k]; a.adam_v[pi + k] = v[k]; }
    }
  }
}

// Accumulator rows of row quarter q: bm = 128 -> rows 32q .. 32q+31 in lanes 0..31;
// bm = 64 -> row m lives in tile lane (m % 16) + 32 * (m / 16): rows 16q .. 16q+15 in the
// quarter's first 16 lanes.
__device__ __forceinline__ int rows_per_quarter(int bm) { return bm == 64 ? 16 : 32; }

// E_OPT: the accumulator tile IS the weight gradient.  Per (row, 4 columns) thread: optimizer on
// the fp32 master (+ moments), bf16 shadow refresh (j.shadow) -- master / moments of this thread's elements
// are fetched BEFORE the accumulator wait, so the update pays no exposed load latency (Adam
// without the prefetch: +4.3 us per step, measured).  fp8 mode: the updated tile is parked in
// the staging buffer and re-quantised one K-group (32 columns of a row) per lane pair, which also
// stores the group's exactly dequantised bf16 values into work_dq (fwd1 / fwd2 read those) or, on
// the last step of a federated round, into the upload shadow (the committee's validation operand),
// just as the e4m3 bytes go to the upload blob instead of the work blob then.  On the last
// step the values (optionally Byzantine-transformed) also go to the upload buffers the committee
// and the FedAvg kernel read.  BM = j.bm: the prefetch holds only the rows the tile has.
template <bool FP8, int BM>
__device__ __forceinline__ void epilogue_opt(const Job& j, const Args& a, int q, int half, int lane,
                                             uint64_t* accum_bar, const wg::AccTile& at, float* stg,
                                             Pipe& pp) {
  constexpr int rpq = BM == 64 ? 16 : 32;        // rows_per_quarter(BM)
  constexpr int n_it = rpq / 4;                  // staged store iterations: 4 rows each
  const int row_base = j.m0 + q * rpq;
  const int cr = lane >> 3, cg = (lane & 7) * 4;
  const int nc = j.n0 + half * 32;               // this warp's 32 columns
  const long long pbase = reinterpret_cast<float*>(j.d) - a.master;
  // row rr of this quarter is accumulator-tile lane 32 q + rr for either tile height (lane128 / lane64)
  const float* gt = at.p + q * 32 * at.pitch + half * 32 + cg;
  // Prefetch ring of kPre row groups: all of a 64-row tile's four; a 128-row tile's eight would not
  // fit the epilogue's registers, so its groups 4..7 are fetched while groups 0..3 are updated.
  constexpr int kPre = n_it < 4 ? n_it : 4;
  float4 wpre[kPre], mpre[kPre], vpre[kPre];
  auto prefetch = [&](int it) {
    const int rw = row_base + it * 4 + cr, col = nc + cg;
    const bool ok = rw < j.M && col + 3 < j.N;
    const long long pi = pbase + static_cast<long long>(rw) * j.ldd + col;
    wpre[it % kPre] = ok ? __ldcg(reinterpret_cast<const float4*>(a.master + pi)) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (a.adam) {
      mpre[it % kPre] = ok ? __ldcg(reinterpret_cast<const float4*>(a.adam_m + pi)) : make_float4(0.f, 0.f, 0.f, 0.f);
      vpre[it % kPre] = ok ? __ldcg(reinterpret_cast<const float4*>(a.adam_v + pi)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
#pragma unroll
  for (int it = 0; it < kPre; ++it) prefetch(it);
  const bool up = j.last && a.has_fed;
  UploadDst ud{};
  if (up) ud = upload_dst<FP8>(a);
  uint8_t* qblob = (FP8 && up) ? ud.blob : a.work_q;
  ptx::mbar_wait(accum_bar, pp.tile & 1);
  ++pp.tile;
  const bool stampit = j.dbg != nullptr && blockIdx.x == 0 && threadIdx.x == kEpiT0;
  if (stampit) j.dbg[j.dbg_slot] = globaltimer_ns();
  {
#pragma unroll
    for (int it = 0; it < n_it; ++it) {
      const int rr = it * 4 + cr, rw = row_base + rr, col = nc + cg;
      const bool valid = rw < j.M && col + 3 < j.N;
      const long long pi = pbase + static_cast<long long>(rw) * j.ldd + col;
      float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
      if (valid) {
        const float4 g = *reinterpret_cast<const float4*>(gt + rr * at.pitch);   // straight from the tile
        w = wpre[it % kPre];
        if (a.adam) {
          float4 m = mpre[it % kPre], s = vpre[it % kPre];
          const float b1 = a.beta1, b2 = a.beta2, c1 = 1.f - a.beta1, c2 = 1.f - a.beta2;
          m.x = b1 * m.x + c1 * g.x; m.y = b1 * m.y + c1 * g.y; m.z = b1 * m.z + c1 * g.z; m.w = b1 * m.w + c1 * g.w;
          s.x = b2 * s.x + c2 * g.x * g.x; s.y = b2 * s.y + c2 * g.y * g.y;
          s.z = b2 * s.z + c2 * g.z * g.z; s.w = b2 * s.w + c2 * g.w * g.w;
          w.x -= a.lr * (m.x / j.bc1) / (sqrtf(s.x / j.bc2) + a.eps);
          w.y -= a.lr * (m.y / j.bc1) / (sqrtf(s.y / j.bc2) + a.eps);
          w.z -= a.lr * (m.z / j.bc1) / (sqrtf(s.z / j.bc2) + a.eps);
          w.w -= a.lr * (m.w / j.bc1) / (sqrtf(s.w / j.bc2) + a.eps);
          *reinterpret_cast<float4*>(a.adam_m + pi) = m;
          *reinterpret_cast<float4*>(a.adam_v + pi) = s;
        } else {
          w.x -= a.lr * g.x; w.y -= a.lr * g.y; w.z -= a.lr * g.z; w.w -= a.lr * g.w;
        }
        *reinterpret_cast<float4*>(a.master + pi) = w;
        if (j.shadow) *reinterpret_cast<uint2*>(a.shadow + pi) = make_uint2(pack2(w.x, w.y), pack2(w.z, w.w));
        if (up) {
          if (ud.global != nullptr) {   // Byzantine client (fault injection, SURVEY.md 5.3)
            const float4 g0 = __ldcg(reinterpret_cast<const float4*>(ud.global + pi));
            w.x = g0.x - ud.byz_scale * (w.x - g0.x); w.y = g0.y - ud.byz_scale * (w.y - g0.y);
            w.z = g0.z - ud.byz_scale * (w.z - g0.z); w.w = g0.w - ud.byz_scale * (w.w - g0.w);
          }
          *reinterpret_cast<float4*>(ud.master + pi) = w;
          if (!FP8) *reinterpret_cast<uint2*>(ud.shadow + pi) = make_uint2(pack2(w.x, w.y), pack2(w.z, w.w));
        }
      }
      // fp8: park the updated values in the staging tile; they are re-quantised row-wise below
      if (FP8) *reinterpret_cast<float4*>(stg + rr * kStgLd + cg) = w;
      if (it + kPre < n_it) prefetch(it + kPre);
    }
    if (FP8) {
      // Two lanes per row of the staged sub-tile: the row's 32 columns are exactly one K-group of
      // the weight matrix; each lane takes 16 of them, one shuffle combines the two halves' amax,
      // and each lane writes its 16 e4m3 bytes and 32 bytes of bf16.  One thread per row (16
      // lanes busy on a 64-row tile) took 2.0 us of the 3.0 us Adam + MXFP8 epilogue, measured;
      // a shuffle-per-4-columns version cost 3.7 us per step.
      __syncwarp();
      const int hh = lane & 1, c0 = hh * 16;
      const int nv = j.N - nc < 32 ? j.N - nc : 32;          // valid columns of this group (multiple of 8)
      const int nh = nv - c0;                                 // valid columns of this lane's half
#pragma unroll
      for (int p = 0; p < rpq; p += 16) {
        const int rr = p + (lane >> 1), rw = row_base + rr;
        float x[16];
        const float4* sp = reinterpret_cast<const float4*>(stg + rr * kStgLd + c0);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float4 t = sp[k];
          x[4 * k] = t.x; x[4 * k + 1] = t.y; x[4 * k + 2] = t.z; x[4 * k + 3] = t.w;
        }
        float amax = 0.f;
#pragma unroll
        for (int k = 0; k < 16; ++k) amax = fmaxf(amax, fabsf(x[k]));
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
        if (rw < j.M && nv > 0) {
          const int e = epi::mx8_scale_byte(amax);
          const float inv = epi::mx8_inv_scale(e);
          uint32_t w4[4];
#pragma unroll
          for (int k = 0; k < 4; ++k)
            w4[k] = epi::mx8_pack4(x[4 * k] * inv, x[4 * k + 1] * inv, x[4 * k + 2] * inv, x[4 * k + 3] * inv);
          // like the blob: the last step of a federated round publishes instead of refreshing the
          // work copies (the next round re-derives them from the new global model)
          uint4* dq = reinterpret_cast<uint4*>(up ? ud.shadow + pbase + static_cast<long long>(rw) * j.ldd + nc + c0
                                                  : a.work_dq + j.dq_off + static_cast<long long>(rw) * j.ldq + nc + c0);
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            if (k * 8 >= nh) break;
            const uint2 lo = epi::mx8_dq4(w4[2 * k], e), hi = epi::mx8_dq4(w4[2 * k + 1], e);
            dq[k] = make_uint4(lo.x, lo.y, hi.x, hi.y);
          }
          if (nh > 0)
            *reinterpret_cast<uint4*>(qblob + j.q_off + static_cast<long long>(rw) * j.ldq + nc + c0) =
                make_uint4(w4[0], w4[1], w4[2], w4[3]);
          if (hh == 0) qblob[j.qsf_off + epi::mx8_sf_index(rw, nc >> 5, j.q_nkb)] = static_cast<uint8_t>(e);
        }
      }
    }
    __syncwarp();
  }
  if (stampit) j.dbg[j.dbg_slot + 1] = globaltimer_ns();
}

// epilogue warps 4..11: q = row quarter, half = which 32 of the tile's 64 columns
template <bool FP8>
__device__ __forceinline__ void epilogue_tile(const Job& j, const Args& a, int q, int half, int lane,
                                              uint64_t* accum_bar, const wg::AccTile& at,
                                              float* stg, float* sbias, Pipe& pp) {
  {
    const int et = threadIdx.x - kEpiT0;
    // coherent (L2) loads: the biases are rewritten by the optimizer phase of this same kernel
    if (et < kBN) sbias[et] = (j.bias != nullptr && j.n0 + et < j.N) ? __ldcg(j.bias + j.n0 + et) : 0.f;
    epi_bar();
  }
  if (j.mode == E_OPT) {
    if (j.bm == 64) epilogue_opt<FP8, 64>(j, a, q, half, lane, accum_bar, at, stg, pp);
    else epilogue_opt<FP8, kBM>(j, a, q, half, lane, accum_bar, at, stg, pp);
    return;
  }
  const int rpq = rows_per_quarter(j.bm);
  const int row_base = j.m0 + q * rpq;
  const int row = row_base + lane;
  const bool row_ok = lane < rpq && row < j.M;
  const int cr = lane >> 3, cg = (lane & 7) * 4;
  const uint32_t taddr = static_cast<uint32_t>(q * 32) << 16;
  ptx::mbar_wait(accum_bar, pp.tile & 1);
  ++pp.tile;
  const bool stampit = j.dbg != nullptr && blockIdx.x == 0 && threadIdx.x == kEpiT0;
  if (stampit) j.dbg[j.dbg_slot] = globaltimer_ns();

  if (j.mode != E_XENT) {
    const int c = half;
    const int nc = j.n0 + c * 32;
    if (nc < j.N) {
      uint32_t r[32];
      wg::acc_ld32(at, taddr + c * 32, r);
      float v[32];
#pragma unroll
      for (int k = 0; k < 32; ++k) v[k] = __uint_as_float(r[k]) + sbias[c * 32 + k];
      if (j.mode == E_BIAS_RELU_BF16) {
#pragma unroll
        for (int k = 0; k < 32; ++k) v[k] = fmaxf(v[k], 0.f);
        if (FP8 && row_ok) {
          // fwd2's A operand: this thread's 32 columns of h are exactly one K-group, quantised
          // to e4m3 and stored dequantised
          uint32_t w[8];
          const int e = epi::mx8_quant32(v, w);
          epi::mx8_dq32_store(w, e, a.h_dq + static_cast<long long>(row) * a.hidden + nc);
        }
      } else if (j.mode == E_MASK_COLSUM_BF16) {
        // coalesced (L2-coherent) load of the mask tile through the staging buffer
#pragma unroll
        for (int it = 0; it < 8; ++it) {
          const int rr = it * 4 + cr, rw = row_base + rr, col = nc + cg;
          float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
          if (rr < rpq && rw < j.M && col + 3 < j.N) {
            const uint2 u = __ldcg(reinterpret_cast<const uint2*>(j.aux + static_cast<long long>(rw) * j.ldd + col));
            const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
            const float2 hi2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
            x = make_float4(lo.x, lo.y, hi2.x, hi2.y);
          }
          *reinterpret_cast<float4*>(stg + rr * kStgLd + cg) = x;
        }
        __syncwarp();
        float m[32];
        stage_get(stg, lane, m);
        __syncwarp();
#pragma unroll
        for (int k = 0; k < 32; ++k) v[k] = m[k] > 0.f ? v[k] : 0.f;
      }
      stage_put(stg, lane, v);
      __syncwarp();
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int rr = it * 4 + cr, rw = row_base + rr, col = nc + cg;
        if (rr >= rpq || rw >= j.M || col >= j.N) continue;
        const float4 x = *reinterpret_cast<const float4*>(stg + rr * kStgLd + cg);
        const long long off = static_cast<long long>(rw) * j.ldd + col;
        if (j.mode == E_F32) {
          float* d = reinterpret_cast<float*>(j.d) + off;
          if (col + 3 < j.N) *reinterpret_cast<float4*>(d) = x;
          else {
            const float xs[4] = {x.x, x.y, x.z, x.w};
            for (int k = 0; k < 4; ++k) if (col + k < j.N) d[k] = xs[k];
          }
        } else {
          __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(j.d) + off;
          *reinterpret_cast<uint2*>(d) = make_uint2(pack2(x.x, x.y), pack2(x.z, x.w));
        }
      }
      if (j.colsum != nullptr) {
        const float tot = col_sum32(stg, lane, min(rpq, j.M - row_base));
        if (nc + lane < j.N) atomicAdd(j.colsum + nc + lane, tot);
      }
      __syncwarp();
    }
  } else if (half == 0) {
    // softmax cross-entropy over the N (<= 64) logits of each row (plan 0 only: general hidden
    // sizes; one thread owns a whole row, the second half of the epilogue warps idles)
    const int32_t label = row_ok ? j.labels[row] : -1;
    float vmax = -INFINITY, zlab = 0.f;
    int amax = -1;
    float z[64];
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      uint32_t r[32];
      wg::acc_ld32(at, taddr + c * 32, r);
#pragma unroll
      for (int k = 0; k < 32; ++k) {
        const int n = c * 32 + k;
        const float x = __uint_as_float(r[k]) + sbias[n];
        z[n] = x;
        if (n < j.N) {
          if (x > vmax) { vmax = x; amax = n; }
          if (n == label) zlab = x;
        }
      }
    }
    float sum = 0.f;
#pragma unroll
    for (int n = 0; n < 64; ++n)
      if (n < j.N) sum += __expf(z[n] - vmax);
    const float inv = 1.f / sum;
    float loss = row_ok ? (__logf(sum) + vmax - zlab) : 0.f;
    const bool hit = row_ok && (amax == label);
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      float (&v)[32] = *reinterpret_cast<float(*)[32]>(z + c * 32);   // dlogits overwrite their logits
#pragma unroll
      for (int k = 0; k < 32; ++k) {
        const int n = c * 32 + k;
        v[k] = (n < j.N && row_ok)
                   ? (__expf(z[n] - vmax) * inv - (n == label ? 1.f : 0.f)) * j.grad_scale
                   : 0.f;
      }
      stage_put(stg, lane, v);
      __syncwarp();
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int rr = it * 4 + cr, rw = row_base + rr, col = c * 32 + cg;
        if (rw >= j.M || col >= j.ldd) continue;
        const float4 x = *reinterpret_cast<const float4*>(stg + rr * kStgLd + cg);
        __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(j.d) + static_cast<long long>(rw) * j.ldd + col;
        *reinterpret_cast<uint2*>(d) = make_uint2(pack2(x.x, x.y), pack2(x.z, x.w));
      }
      if (j.colsum != nullptr) {
        const float tot = col_sum32(stg, lane, 32);
        if (c * 32 + lane < j.N) atomicAdd(j.colsum + c * 32 + lane, tot);
      }
      __syncwarp();
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, off);
    const unsigned cnt = __popc(__ballot_sync(0xffffffffu, hit));
    if (lane == 0) {
      atomicAdd(a.loss_sum, loss);
      if (cnt) atomicAdd(a.correct, cnt);
    }
  }
  if (stampit) j.dbg[j.dbg_slot + 1] = globaltimer_ns();
}

// bit e set <=> bf16 element e of the 8 in u is > 0 (sign clear and not zero); in fp8 mode the
// dequantised h_dq is > 0 exactly where the e4m3 h is
__device__ __forceinline__ uint32_t pos_mask8(const uint4 u) {
  const uint32_t wds[4] = {u.x, u.y, u.z, u.w};
  uint32_t m = 0u;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    m |= (((wds[e] & 0xFFFFu) != 0u && (wds[e] & 0x8000u) == 0u) ? 1u : 0u) << (e * 2);
    m |= (((wds[e] >> 16) != 0u && (wds[e] & 0x80000000u) == 0u) ? 1u : 0u) << (e * 2 + 1);
  }
  return m;
}

// Thread layout of the chain epilogues (fwd1 of plan 4, E1-E3) on a BM x 64 tile: epilogue warp w
// (0..7) owns rows BM/8 * w .. +BM/8, so all the threads of a row sit in one warp and combine by
// shuffles.  Lane l takes row BM/8 * w + l % (BM/8) and column group l / (BM/8) of 64 / TPR
// columns, TPR = 256 / BM threads per row: 2 x 32 columns at BM = 128, 4 x 16 at BM = 64.  The
// other threads of lane l's row are lane l ^ 16 and, at BM = 64, lanes l ^ 8 and l ^ 24;
// consecutive lanes take consecutive rows, which keeps the accumulator-tile reads and the
// swizzled 16-byte stores free of bank conflicts.
template <int BM>
struct ChainThread {
  static constexpr int kRpw = BM / 8, kTpr = 32 / kRpw, kCpt = 64 / kTpr;
  int rl, c;   // row inside the tile, column group
  const float* acc;   // the row in the accumulator tile
  __device__ __forceinline__ ChainThread(const wg::AccTile& at, int lane) {
    rl = kRpw * ((static_cast<int>(threadIdx.x) - kEpiT0) >> 5) + lane % kRpw;
    c = lane / kRpw;
    acc = at.p + (BM == 64 ? lane64(rl) : lane128(rl)) * at.pitch;
  }
};

// Column sums of the [BM][kRedLd] fp32 tile `red` the epilogue threads have just written: after an
// epi_bar, thread t sums rows 32 (t / 64) .. +32 of column t % 64 into dst[col] (col < n).  Every
// atomic adds the sum of 32 batch rows rounded as epi::col_sum32 rounds it, at either tile height,
// so the bias gradients differ between plans only by the order of the atomics.
template <int BM>
__device__ __forceinline__ void red_colsum(const float* red, float* dst, int n) {
  epi_bar();
  const int et = threadIdx.x - kEpiT0, col = et & 63, r0 = (et >> 6) * 32;
  if (r0 >= BM) return;
  float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int rr = 0; rr < 32; ++rr) t[rr & 3] += red[(r0 + rr) * kRedLd + col];
  if (col < n) atomicAdd(dst + col, (t[0] + t[1]) + (t[2] + t[3]));
}

// DP-SGD: the same 32-row column sums, each stored to its own workspace slot (row group r0 / 32 of the
// tile at dst + (r0 / 32) kDpWsLd) instead of added: the bias CTA sums the slots in a fixed order.
template <int BM>
__device__ __forceinline__ void red_colsum_ws(const float* red, float* dst) {
  epi_bar();
  const int et = threadIdx.x - kEpiT0, col = et & 63, r0 = (et >> 6) * 32;
  if (r0 >= BM) return;
  float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int rr = 0; rr < 32; ++rr) t[rr & 3] += red[(r0 + rr) * kRedLd + col];
  dst[(r0 / 32) * kDpWsLd + col] = (t[0] + t[1]) + (t[2] + t[3]);
}
__device__ __forceinline__ void st_cluster_f4(uint32_t addr, float4 v) {
  asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w) : "memory");
}
__device__ __forceinline__ float bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
// k_scale_rows' rule: bf16(v c), exactly +0 where c is +-0
__device__ __forceinline__ float dp_scaled(float v, float c) {
  return (__float_as_uint(c) & 0x7FFFFFFFu) == 0u ? 0.f : bf16_round(so_mul(v, c));
}

// Plan 4: fwd1 epilogue of chain CTA `slice` (cluster rank) of a 64-row M-tile.  Its 64 x 64 tile
// of h is K-block `slice` of fwd2's A operand in all four CTAs of the cluster: each thread stores
// its 16 columns of one row (ChainThread<64>) -- bf16 h, or in fp8 mode the exactly dequantised
// e4m3 h, the bytes plan 3's TMA loads from h / h_dq -- into the swizzled local h tile; one thread
// then bulk-copies the 8 KB slice to the same offset of the three peers.  Returns the relu mask of
// these 16 columns, which are exactly the ones the thread owns in chain step E3.
//   * An MXFP8 group (32 columns) spans the lane pair l, l ^ 8: one shuffle combines its amax, so
//     the scale byte and the e4m3 bytes are those of epi::mx8_quant32 on the whole group.
//   * The h tile overlays the fwd1 ring: the local slice waits for this CTA's ring (drained before
//     accum_bar), the copies for ring_free (all four rings drained).
//   * The accumulator tile is overwritten by fwd2 once hx completes, and hx's only arrive follows
//     the epi_bar that every epilogue thread reaches after its accumulator reads.
//   * The copies read this CTA's slice until the peers' hx complete: chain step E3 stages dh in
//     a received slice instead.  They have all landed by the grid barrier after the chain.
//   * The global bf16 h is still stored (dW2 reads it in phase B); the global h_dq has no reader.
//   * DP-SGD (pdp): the row's ||h||^2 over this slice's 64 bf16 columns and ||x||^2 over a quarter of x's
//     8-column chunks (chunk k on slice k % 4; global, L2-resident since fwd1's TMA), summed over the
//     row's four threads and parked in this CTA's own partials (kOffDpOwn) for the chain's exchange.
template <bool FP8, bool DP = false>
__device__ __forceinline__ uint32_t fwd1_epilogue_x(const Job& j, const Args& a, uint8_t* smem, const ChainBars& cb,
                                                    int lane, uint64_t* accum_bar, const wg::AccTile& at,
                                                    float* sbias, Pipe& pp, uint32_t par, int slice,
                                                    const TrainerDp* pdp = nullptr) {
  const int et = threadIdx.x - kEpiT0;
  if (et < kBN) sbias[et] = __ldcg(j.bias + j.n0 + et);   // the optimizer of this kernel rewrites b1
  epi_bar();
  const ChainThread<kBMx> th(at, lane);
  const int row = j.m0 + th.rl, c0 = th.c * 16;
  const bool row_ok = row < j.M;
  const bool stampit = j.dbg != nullptr && blockIdx.x == 0 && threadIdx.x == kEpiT0;
  ptx::mbar_wait(accum_bar, pp.tile & 1);
  ++pp.tile;
  if (stampit) j.dbg[j.dbg_slot] = globaltimer_ns();
  float v[16];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float4 t = reinterpret_cast<const float4*>(th.acc + c0)[k];
    v[4 * k] = fmaxf(t.x + sbias[c0 + 4 * k], 0.f);
    v[4 * k + 1] = fmaxf(t.y + sbias[c0 + 4 * k + 1], 0.f);
    v[4 * k + 2] = fmaxf(t.z + sbias[c0 + 4 * k + 2], 0.f);
    v[4 * k + 3] = fmaxf(t.w + sbias[c0 + 4 * k + 3], 0.f);
  }
  uint4 hb[2];   // bf16 h: the global copy, and in bf16 mode also fwd2's operand
#pragma unroll
  for (int jj = 0; jj < 2; ++jj)
    hb[jj] = make_uint4(pack2(v[8 * jj], v[8 * jj + 1]), pack2(v[8 * jj + 2], v[8 * jj + 3]),
                        pack2(v[8 * jj + 4], v[8 * jj + 5]), pack2(v[8 * jj + 6], v[8 * jj + 7]));
  uint4 hv[2] = {hb[0], hb[1]};
  if (FP8) {
    float amax = 0.f;
#pragma unroll
    for (int k = 0; k < 16; ++k) amax = fmaxf(amax, fabsf(v[k]));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 8));   // the group's other 16 columns
    const int e = epi::mx8_scale_byte(amax);
    const float inv = epi::mx8_inv_scale(e);
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      const float* x = v + 8 * jj;
      const uint2 lo = epi::mx8_dq4(epi::mx8_pack4(x[0] * inv, x[1] * inv, x[2] * inv, x[3] * inv), e);
      const uint2 hi = epi::mx8_dq4(epi::mx8_pack4(x[4] * inv, x[5] * inv, x[6] * inv, x[7] * inv), e);
      hv[jj] = make_uint4(lo.x, lo.y, hi.x, hi.y);
    }
  }
  uint32_t mk = 0u;
#pragma unroll
  for (int jj = 0; jj < 2; ++jj) {
    if (!row_ok) hv[jj] = make_uint4(0u, 0u, 0u, 0u);   // rows past the batch: zero, as the TMA fills them
    mk |= pos_mask8(hv[jj]) << (jj * 8);
  }
  // this CTA's own ring is drained (the MMA released its last stage before accum_bar)
  uint8_t* hs = smem + kOffH + slice * kHSlice;
#pragma unroll
  for (int jj = 0; jj < 2; ++jj) st_sw128(hs, th.rl, 2 * th.c + jj, hv[jj]);
  ptx::fence_proxy_async_smem();   // -> the local wgmma and the bulk copies (async proxy)
  epi_bar();                       // slice complete; every accumulator and sbias read done
  if (threadIdx.x == kEpiT0) {
    const uint32_t hxa = ptx::smem_u32(cb.hx);
    ptx::mbar_expect_tx(cb.hx, (kCluster - 1) * kHSlice);   // own slice here; expect the three peers'
    ptx::mbar_wait_cluster(cb.ring_free, par);
    for (uint32_t r = 1; r < kCluster; ++r) {
      const uint32_t peer = (slice + r) % kCluster;
      ptx::bulk_s2cluster(ptx::mapa(ptx::smem_u32(hs), peer), hs, kHSlice, ptx::mapa(hxa, peer));
    }
  }
  if (stampit) j.dbg[1] = globaltimer_ns();
  if (row_ok) {   // a warp's two stores cover its 8 rows x 128 bytes
    uint4* d = reinterpret_cast<uint4*>(a.h + static_cast<long long>(row) * j.ldd + j.n0 + c0);
    d[0] = hb[0];
    d[1] = hb[1];
  }
  if constexpr (DP) {
    float hs = 0.f, xs = 0.f;
    if (row_ok) {
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const uint32_t wds[4] = {hb[jj].x, hb[jj].y, hb[jj].z, hb[jj].w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&wds[e]));
          hs = fmaf(f.x, f.x, hs);
          hs = fmaf(f.y, f.y, hs);
        }
      }
      const uint4* xr = reinterpret_cast<const uint4*>(pdp->x + static_cast<long long>(j.a_c1 + th.rl) * a.in_dim);
      for (int k = slice + 4 * th.c; k < a.in_dim / 8; k += 16) {
        const uint4 u = __ldcg(xr + k);
        const uint32_t wds[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&wds[e]));
          xs = fmaf(f.x, f.x, xs);
          xs = fmaf(f.y, f.y, xs);
        }
      }
    }
    // the row's four threads are lanes l ^ 8, l ^ 16: every one ends with the same sums
    hs += __shfl_xor_sync(0xffffffffu, hs, 8);
    xs += __shfl_xor_sync(0xffffffffu, xs, 8);
    hs += __shfl_xor_sync(0xffffffffu, hs, 16);
    xs += __shfl_xor_sync(0xffffffffu, xs, 16);
    if (th.c == 0) reinterpret_cast<float2*>(smem + kOffDpOwn)[th.rl] = make_float2(hs, xs);
  }
  if (stampit) j.dbg[j.dbg_slot + 1] = globaltimer_ns();
  return mk;
}

// ---------------------------------------------------------------- fused chain of one M-tile
//   (BM = 128 rows in plan 3, 64 in plan 4; h was produced by P1 and arrives by TMA: bf16, or in
//    fp8 mode the dequantised e4m3 h_dq; plan 4: straight from the cluster's fwd1 epilogues)
//   fwd2  logits[BM x 64] = h W2^T           (A, B from smem)             -> accumulator tile
//   E2    softmax-xent per row -> dlogits -> smem (dh's A operand) + global
//   dh    acc[BM x 64 slice] = dlogits W2    (B = W2 MN-major)            -> accumulator tile
//         (written once every epilogue thread has read its logits: dl_ready)
//   E3    dh = acc * relu'(h) -> bf16 global, db1
// logits / dlogits never make the global -> TMA round trip; the three GEMMs cost one grid barrier.
// Four CTAs per M-tile: all redo the cheap fwd2 + xent so that the dh GEMM and its epilogue run
// 4-wide (64 hidden columns each); loss, db2 and the global dlogits copy are done by one of them.
// with_h = false (plan 4): the h tile arrives from the cluster's fwd1 epilogues instead; with_h is
// plan 3's 128-row tile, two 64-row boxes per K-block
__device__ __forceinline__ void chain_produce(const Maps& maps, uint8_t* smem, const ChainBars& cb, int m0,
                                              int slice, bool with_h) {
  if (ptx::elect_one()) {
    ptx::mbar_expect_tx(cb.w2k, 32768);
    if (with_h) ptx::mbar_expect_tx(cb.h, 65536);
    ptx::mbar_expect_tx(cb.w2mn, 8192);
    // in the order the chain consumes them: h and W2 (fwd2) first, W2^T (dh) last
    if (with_h) {
#pragma unroll
      for (int kb = 0; kb < 4; ++kb) {
        ptx::tma_load_3d(smem + kOffH + kb * 16384, &maps.h_k, cb.h, kb * 64, m0, 0);
        ptx::tma_load_3d(smem + kOffH + kb * 16384 + 8192, &maps.h_k, cb.h, kb * 64, m0 + 64, 0);
      }
    }
#pragma unroll
    for (int kb = 0; kb < 4; ++kb)
      ptx::tma_load_3d(smem + kOffW2K + kb * 8192, &maps.w2_k, cb.w2k, kb * 64, 0, 0);
    ptx::tma_load_3d(smem + kOffW2MN, &maps.w2_mn, cb.w2mn, slice * 64, 0, 0);
  }
  __syncwarp();
}

template <int BM>
__device__ __forceinline__ void chain_mma(uint8_t* smem, const ChainBars& cb, const wg::AccTile& at, uint32_t par,
                                          bool fused) {
  constexpr bool two = BM == kBM;            // two m64 halves per k16
  constexpr uint32_t kb_bytes = BM * 128u;   // one K-block of the h tile
  const uint32_t base = ptx::smem_u32(smem);
  // fwd2: BM x 64 x 256, A = h (TMA, or plan 4: stored by the cluster's fwd1 epilogues), B = W2 K-major
  ptx::mbar_wait(cb.w2k, par);
  if (fused) {
    ptx::mbar_wait_cluster(cb.hx, par);
    ptx::fence_proxy_async_smem();   // the peers' st.async data -> this warpgroup's wgmma (async proxy)
  } else {
    ptx::mbar_wait(cb.h, par);
  }
  float l0[32], l1[32];
  wg::zero(l0);
  wg::zero(l1);
  const uint32_t ha = base + kOffH, wb = base + kOffW2K;
  wg::fence();
#pragma unroll
  for (uint32_t kb = 0; kb < 4; ++kb)
#pragma unroll
    for (uint32_t k = 0; k < 4; ++k) {
      const uint64_t bd = wg::desc(wb + kb * 8192u + k * 32u, 16);
      wg::mma_bf16<64, 0, 0>(l0, wg::desc(ha + kb * kb_bytes + k * 32u, 16), bd, (kb > 0 || k > 0) ? 1u : 0u);
      if (two)
        wg::mma_bf16<64, 0, 0>(l1, wg::desc(ha + kb * kb_bytes + 8192u + k * 32u, 16), bd, (kb > 0 || k > 0) ? 1u : 0u);
    }
  wg::commit();
  wg::wait<0>();
  wg::reg_fence(l0);
  if (two) {
    wg::reg_fence(l1);
    wg::acc_put<64>(at, 0, l0, lane128);
    wg::acc_put<64>(at, 0, l1, lane128_hi);
  } else {
    wg::acc_put<64>(at, 0, l0, lane64);
  }
  ptx::mbar_arrive(cb.acc_l);
  // dh: BM x 64 x 64, A = dlogits (smem, written by the epilogue warps), B = W2 MN-major slice
  ptx::mbar_wait(cb.w2mn, par);
  ptx::mbar_wait(cb.dl_ready, par);
  wg::zero(l0);
  wg::zero(l1);
  wg::fence();
#pragma unroll
  for (uint32_t k = 0; k < 4; ++k) {
    const uint64_t bd = wg::desc(base + kOffW2MN + k * 2048u, 8192);
    wg::mma_bf16<64, 0, 1>(l0, wg::desc(base + kOffDL + k * 32u, 16), bd, k > 0);
    if (two) wg::mma_bf16<64, 0, 1>(l1, wg::desc(base + kOffDL + 8192u + k * 32u, 16), bd, k > 0);
  }
  wg::commit();
  wg::wait<0>();
  wg::reg_fence(l0);
  if (two) {
    wg::reg_fence(l1);
    wg::acc_put<64>(at, 0, l0, lane128);
    wg::acc_put<64>(at, 0, l1, lane128_hi);
  } else {
    wg::acc_put<64>(at, 0, l0, lane64);
  }
  ptx::mbar_arrive(cb.acc_dh);
}

// Epilogue of the chain on a BM-row M-tile, thread layout ChainThread<BM>: each thread owns one row
// rl and, in E1 / E3, the 64 / TPR hidden columns [cpt c, +cpt) of this CTA's 64-column dh slice.
// E2 splits a row's logits so that the sum of exponentials rounds as one serial scan does (below);
// the threads of a row combine their partials with shuffles.  db1 / db2 are column sums through
// the fp32 tile `red` (the staging buffers) and one atomic per column and 32 rows (red_colsum).
//
// DP-SGD (DP, plan 4; pdp, px the exchange mbarrier): E2 also forms ||dz||^2 of the row and leaves the
// dlogits store and db2 to E3, which needs c.  E3 forms ||dh||^2 over this slice, sends the row's
// three slice partials to all four CTAs of the cluster (px), sums the four slices in slice order 0..3 --
// so every CTA computes the same bits of c -- and then scales and stores dh (and dz', db2 on slices 2
// and 1), with the bias column sums in the workspace.
template <int BM, bool DP = false>
__device__ __forceinline__ void chain_epilogue(const Args& a, uint8_t* smem, const ChainBars& cb,
                                               const wg::AccTile& at, int lane, float* red, float* sb,
                                               uint32_t par, int m0, int r0, int slice,
                                               unsigned long long* dbg, bool fused, uint32_t mk_fused,
                                               const TrainerDp* pdp = nullptr, uint64_t* px = nullptr,
                                               int step = 0) {
  static_assert(!DP || BM == kBMx, "DP-SGD runs in plan 4");
  using TH = ChainThread<BM>;
  constexpr int kTpr = TH::kTpr, kCpt = TH::kCpt;
  auto stampc = [&](int slot) {
    if (dbg != nullptr && blockIdx.x == 0 && threadIdx.x == kEpiT0) dbg[slot] = globaltimer_ns();
  };
  const TH th(at, lane);
  const int rl = th.rl;                // row inside the tile
  const int row = m0 + rl;             // row inside the mini-batch
  const bool row_ok = row < a.B;
  const int32_t label = row_ok ? __ldg(a.labels + r0 + row) : -1;   // issued early: needed by E2
  const int C = a.n_classes;
  const int et = threadIdx.x - kEpiT0;
  {
    // coherent loads: the optimizer of this kernel rewrites the biases
    sb[et] = __ldcg(a.b1 + et);        // kEpiThreads == kChainH == 256
    if (et < 64) sb[kChainH + et] = et < C ? __ldcg(a.b2 + et) : 0.f;
    epi_bar();
  }
  const int rw0 = TH::kRpw * (et >> 5);   // first row of this warp

  // ---- E1: relu mask of this thread's hidden columns [64 slice + cpt c, +cpt), read back
  //          through the swizzle from the h tile the TMA dropped into the A-operand slots (fp8:
  //          h_dq > 0 exactly where the e4m3 h is)
  //          plan 4 (fused): the fwd1 epilogue built the mask from the same values in registers
  uint32_t mk = mk_fused;
  if (!fused) {
    ptx::mbar_wait(cb.h, par);
    stampc(6);
    const uint8_t* hs = smem + kOffH + slice * (BM * 128);
#pragma unroll
    for (int jj = 0; jj < kCpt / 8; ++jj)
      mk |= pos_mask8(epi::ld_sw128(hs, rl, th.c * (kCpt / 8) + jj)) << (jj * 8);
  } else if (dbg != nullptr && blockIdx.x == 0 && threadIdx.x == kEpiT0) {
    ptx::mbar_wait_cluster(cb.hx, par);   // stamp only: the whole h tile has landed here
    stampc(6);
  }
  stampc(7);

  float dz2 = 0.f;   // DP-SGD: ||dz||^2 of the row's bf16 dlogits
  // ---- E2: softmax cross-entropy of the row.  Logit n = 32 hh + 4 i + j (i = 0..7) of half hh
  //          is summed into partial ps[j], and the row's sum is ((ps0 + ps1) + (ps2 + ps3)) of half 0
  //          plus that of half 1.  A thread owns one half and NJ = 8 / TPR of the residues j:
  //          TPR = 2 -> all four, TPR = 4 -> {0, 1} or {2, 3}, so that with exact maxima and
  //          products both tile heights produce the same dlogits bits.
  ptx::mbar_wait(cb.acc_l, par);
  stampc(8);
  {
    constexpr int NJ = 8 / kTpr;
    const int hh = th.c / (kTpr / 2), j0 = (th.c % (kTpr / 2)) * NJ;
    const int nb = 32 * hh + j0;   // column of z[0]; z[NJ i + jj] is column nb + 4 i + jj
    float z[8 * NJ];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float* src = th.acc + nb + 4 * i;
      if constexpr (NJ == 4) {
        const float4 t = *reinterpret_cast<const float4*>(src);
        z[4 * i] = t.x; z[4 * i + 1] = t.y; z[4 * i + 2] = t.z; z[4 * i + 3] = t.w;
      } else {
        const float2 t = *reinterpret_cast<const float2*>(src);
        z[2 * i] = t.x; z[2 * i + 1] = t.y;
      }
#pragma unroll
      for (int jj = 0; jj < NJ; ++jj) z[NJ * i + jj] += sb[kChainH + nb + 4 * i + jj];
    }
    float vmax = -INFINITY, zlab = 0.f;
    int amax = -1;
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int jj = 0; jj < NJ; ++jj) {   // increasing column: the first maximum wins
        const int n = nb + 4 * i + jj;
        const float x = z[NJ * i + jj];
        if (n < C) {
          if (x > vmax) { vmax = x; amax = n; }
          if (n == label) zlab = x;
        }
      }
    // the row's other threads: lane ^ 16 (the other half) and, at TPR = 4, lane ^ 8 (the other
    // residues of this half); ties go to the lower column, as in a serial scan
#pragma unroll
    for (int off = (kTpr == 4 ? 8 : 16); off <= 16; off <<= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, vmax, off);
      const int oi = __shfl_xor_sync(0xffffffffu, amax, off);
      if (ov > vmax || (ov == vmax && oi >= 0 && (amax < 0 || oi < amax))) { vmax = ov; amax = oi; }
      zlab += __shfl_xor_sync(0xffffffffu, zlab, off);
    }
    stampc(12);
    float ps[NJ];
#pragma unroll
    for (int jj = 0; jj < NJ; ++jj) ps[jj] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i)   // z <- exp(z - max): each exponential is evaluated once
#pragma unroll
      for (int jj = 0; jj < NJ; ++jj) {
        float& x = z[NJ * i + jj];
        x = nb + 4 * i + jj < C ? __expf(x - vmax) : 0.f;
        ps[jj] += x;
      }
    float psum;
    if constexpr (NJ == 4) {
      psum = (ps[0] + ps[1]) + (ps[2] + ps[3]);
    } else {
      psum = ps[0] + ps[1];
      psum += __shfl_xor_sync(0xffffffffu, psum, 8);
    }
    const float sum = psum + __shfl_xor_sync(0xffffffffu, psum, 16);
    const float inv = 1.f / sum;
    const float gs = 1.f / static_cast<float>(a.B);
    // the 4 slice-CTAs of an M-tile all need dlogits in smem, but the bookkeeping is done once:
    const bool do_colsum = !DP && slice == 1, do_global = !DP && slice == 2, do_loss = slice == 3;
    uint8_t* dls = smem + kOffDL;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float v[NJ];
#pragma unroll
      for (int jj = 0; jj < NJ; ++jj) {
        const int n = nb + 4 * i + jj;
        v[jj] = (n < C && row_ok) ? (z[NJ * i + jj] * inv - (n == label ? 1.f : 0.f)) * gs : 0.f;
        if constexpr (DP) {
          const float r = bf16_round(v[jj]);
          dz2 = fmaf(r, r, dz2);
        }
      }
      const int col = nb + 4 * i;
      uint8_t* d = dls + rl * 128 + (((col >> 3) ^ (rl & 7)) << 4) + (col & 7) * 2;
      if constexpr (NJ == 4) {
        *reinterpret_cast<uint2*>(d) = make_uint2(pack2(v[0], v[1]), pack2(v[2], v[3]));
        if (do_colsum) *reinterpret_cast<float4*>(red + rl * kRedLd + col) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
        *reinterpret_cast<uint32_t*>(d) = pack2(v[0], v[1]);
        if (do_colsum) *reinterpret_cast<float2*>(red + rl * kRedLd + col) = make_float2(v[0], v[1]);
      }
    }
    if constexpr (DP) {   // the row's other threads (TPR = 4: lanes l ^ 8, l ^ 16)
      dz2 += __shfl_xor_sync(0xffffffffu, dz2, 8);
      dz2 += __shfl_xor_sync(0xffffffffu, dz2, 16);
    }
    // hand the tile to the dh MMA first, then finish the bookkeeping underneath it
    stampc(13);
    ptx::fence_proxy_async_smem();
    ptx::mbar_arrive(cb.dl_ready);
    stampc(14);
    if (do_colsum) red_colsum<BM>(red, a.gb2, C);
    // dlogits -> global for dW2, read back out of the swizzled tile: this warp wrote its rows whole,
    // and each store instruction covers 4 rows x 128 bytes
    __syncwarp();
    if (do_global) {
#pragma unroll
      for (int it = 0; it < TH::kRpw / 4; ++it) {
        const int rt = rw0 + 4 * it + (lane >> 3), ch = lane & 7;
        const uint4 u = epi::ld_sw128(dls, rt, ch);
        if (m0 + rt < a.B && ch * 8 < a.ncp)
          *reinterpret_cast<uint4*>(a.dlogits + static_cast<long long>(m0 + rt) * a.ncp + ch * 8) = u;
      }
    }
    if (do_loss) {
      const bool own = th.c == 0 && row_ok;   // one thread per row
      float loss = own ? (__logf(sum) + vmax - zlab) : 0.f;
      const bool hit = own && (amax == label);
#pragma unroll
      for (int off = 16; off >= 1; off >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, off);
      const unsigned cnt = __popc(__ballot_sync(0xffffffffu, hit));
      if (lane == 0) {
        atomicAdd(a.loss_sum, loss);
        if (cnt) atomicAdd(a.correct, cnt);
      }
    }
    if (do_colsum) epi_bar();   // every db2 read of `red` done before E3 rewrites it
  }
  stampc(9);

  // ---- E3: dh = (dlogits W2) * relu'(h), db1 -- cpt hidden columns per thread
  ptx::mbar_wait(cb.acc_dh, par);
  stampc(10);
  if constexpr (DP) {
    const TrainerDp& d = *pdp;
    uint8_t* ds = smem + kOffH + ((slice + 1) % kCluster) * kHSlice;   // as below
    const int c0 = th.c * kCpt;
    float vb[kCpt];   // this thread's bf16 dh, as the plain path stores it
    float dh2 = 0.f;
#pragma unroll
    for (int k4 = 0; k4 < kCpt / 4; ++k4) {
      const float4 t = *reinterpret_cast<const float4*>(th.acc + c0 + 4 * k4);
      const float tv[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int b = 4 * k4 + q;
        vb[b] = bf16_round(((mk >> b) & 1u) ? tv[q] : 0.f);
        dh2 = fmaf(vb[b], vb[b], dh2);
      }
    }
    dh2 += __shfl_xor_sync(0xffffffffu, dh2, 8);
    dh2 += __shfl_xor_sync(0xffffffffu, dh2, 16);
    // the exchange: slot [slice][row] of every CTA of the cluster <- (||h||^2, ||x||^2, ||dh||^2) of this slice
    const float4* xb = reinterpret_cast<const float4*>(smem + kOffDpX);
    if (th.c == 0) {
      const float2 own = reinterpret_cast<const float2*>(smem + kOffDpOwn)[rl];
      const uint32_t dst = ptx::smem_u32(xb + slice * 64 + rl);
#pragma unroll
      for (uint32_t r = 0; r < kCluster; ++r) st_cluster_f4(ptx::mapa(dst, r), make_float4(own.x, own.y, dh2, 0.f));
      // each writer releases its own stores to every CTA of the cluster (64 rows x 4 CTAs arrive per phase)
      for (uint32_t r = 0; r < kCluster; ++r) ptx::mbar_arrive_cluster(px, r);
    }
    ptx::mbar_wait_cluster(px, par);
    float hh = 0.f, xx = 0.f, dd = 0.f;
#pragma unroll
    for (int s4 = 0; s4 < kCluster; ++s4) {
      const float4 p = xb[s4 * 64 + rl];
      hh = so_add(hh, p.x); xx = so_add(xx, p.y); dd = so_add(dd, p.z);
    }
    const float b0 = so_add(hh, 1.f), b1 = so_add(xx, 1.f);
    const float sq0 = so_mul(dz2, b0), sq1 = so_mul(dd, b1);
    const float ab0 = so_mul(so_sqrt(dz2), so_sqrt(b0)), ab1 = so_mul(so_sqrt(dd), so_sqrt(b1));
    bool drop = false;
    const float cf = row_ok ? dpsgd_clip_factor(so_add(so_add(0.f, sq0), sq1), so_add(so_add(0.f, ab0), ab1),
                                                d.bsz, d.clip, &drop)
                            : 0.f;
    float* sc = reinterpret_cast<float*>(smem + kOffDpC);
    if (th.c == 0) {
      sc[rl] = cf;
      if (slice == 0 && row_ok) {
        if (drop) atomicAdd(d.dropped, 1);
        if (d.dbg != nullptr) {
          float* o = d.dbg + static_cast<long long>(step) * 5 * a.B + row;
          o[0] = sq0; o[a.B] = sq1; o[2 * a.B] = ab0; o[3 * a.B] = ab1; o[4 * a.B] = cf;
        }
      }
    }
#pragma unroll
    for (int jj = 0; jj < kCpt / 8; ++jj) {
      float v[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) v[q] = dp_scaled(vb[8 * jj + q], cf);
      *reinterpret_cast<float4*>(red + rl * kRedLd + c0 + 8 * jj) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(red + rl * kRedLd + c0 + 8 * jj + 4) = make_float4(v[4], v[5], v[6], v[7]);
      st_sw128(ds, rl, th.c * (kCpt / 8) + jj,
               make_uint4(pack2(v[0], v[1]), pack2(v[2], v[3]), pack2(v[4], v[5]), pack2(v[6], v[7])));
    }
    // a dropped example's h row (which may be what is not finite) is zeroed in the h that dW2 reads
    if (row_ok && (__float_as_uint(cf) & 0x7FFFFFFFu) == 0u) {
      uint4* hp = reinterpret_cast<uint4*>(a.h + static_cast<long long>(row) * a.hidden + slice * 64 + c0);
#pragma unroll
      for (int k = 0; k < kCpt / 8; ++k) hp[k] = make_uint4(0u, 0u, 0u, 0u);
    }
    float* ws = d.bias_ws + static_cast<long long>(m0 / BM) * 2 * kDpWsLd;
    red_colsum_ws<BM>(red, ws + slice * 64);   // its epi_bar also orders the ds reads and sc below
#pragma unroll
    for (int it = 0; it < TH::kRpw / 4; ++it) {
      const int rt = rw0 + 4 * it + (lane >> 3), ch = lane & 7;
      const uint4 u = epi::ld_sw128(ds, rt, ch);
      if (m0 + rt < a.B)
        *reinterpret_cast<uint4*>(a.dh + static_cast<long long>(m0 + rt) * a.hidden + slice * 64 + ch * 8) = u;
    }
    const uint8_t* dls = smem + kOffDL;   // the unscaled bf16 dlogits (the dh MMA has retired)
    auto scale8 = [&](uint4 u, float cr, float* v) {
      const uint32_t wds[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&wds[e]));
        v[2 * e] = dp_scaled(f.x, cr);
        v[2 * e + 1] = dp_scaled(f.y, cr);
      }
    };
    if (slice == 1) {   // db2: column sums of the row's dz' (its 16 columns)
      epi_bar();        // every read of red by the db1 sums is done
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        float v[8];
        scale8(epi::ld_sw128(dls, rl, 2 * th.c + jj), cf, v);
        *reinterpret_cast<float4*>(red + rl * kRedLd + 16 * th.c + 8 * jj) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4*>(red + rl * kRedLd + 16 * th.c + 8 * jj + 4) = make_float4(v[4], v[5], v[6], v[7]);
      }
      red_colsum_ws<BM>(red, ws + kChainH);
    } else if (slice == 2) {   // dz' -> global for dW2
#pragma unroll
      for (int it = 0; it < TH::kRpw / 4; ++it) {
        const int rt = rw0 + 4 * it + (lane >> 3), ch = lane & 7;
        float v[8];
        scale8(epi::ld_sw128(dls, rt, ch), sc[rt], v);
        if (m0 + rt < a.B && ch * 8 < a.ncp)
          *reinterpret_cast<uint4*>(a.dlogits + static_cast<long long>(m0 + rt) * a.ncp + ch * 8) =
              make_uint4(pack2(v[0], v[1]), pack2(v[2], v[3]), pack2(v[4], v[5]), pack2(v[6], v[7]));
      }
    }
  } else {
    // The h tile at kOffH is dead (fwd2 retired before acc_l, the mask is in registers): its first
    // BM x 128 bytes become a bf16 staging tile so that dh leaves the SM 4 rows x 128 bytes per
    // store instruction.  Plan 4: a slice another CTA sent here (it has landed), not this CTA's
    // own, which its bulk copies may still be reading.
    uint8_t* ds = smem + kOffH + (fused ? ((slice + 1) % kCluster) * kHSlice : 0);
    const int c0 = th.c * kCpt;
#pragma unroll
    for (int jj = 0; jj < kCpt / 8; ++jj) {
      float v[8];
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const float4 t = *reinterpret_cast<const float4*>(th.acc + c0 + 8 * jj + 4 * h2);
        const int b = 8 * jj + 4 * h2;
        v[4 * h2] = ((mk >> b) & 1u) ? t.x : 0.f;
        v[4 * h2 + 1] = ((mk >> (b + 1)) & 1u) ? t.y : 0.f;
        v[4 * h2 + 2] = ((mk >> (b + 2)) & 1u) ? t.z : 0.f;
        v[4 * h2 + 3] = ((mk >> (b + 3)) & 1u) ? t.w : 0.f;
        *reinterpret_cast<float4*>(red + rl * kRedLd + c0 + b) = make_float4(v[4 * h2], v[4 * h2 + 1],
                                                                             v[4 * h2 + 2], v[4 * h2 + 3]);
      }
      st_sw128(ds, rl, th.c * (kCpt / 8) + jj,
               make_uint4(pack2(v[0], v[1]), pack2(v[2], v[3]), pack2(v[4], v[5]), pack2(v[6], v[7])));
    }
    red_colsum<BM>(red, a.gb1 + slice * 64, 64);   // its epi_bar also orders the ds reads below
#pragma unroll
    for (int it = 0; it < TH::kRpw / 4; ++it) {
      const int rt = rw0 + 4 * it + (lane >> 3), ch = lane & 7;
      const uint4 u = epi::ld_sw128(ds, rt, ch);
      if (m0 + rt < a.B)
        *reinterpret_cast<uint4*>(a.dh + static_cast<long long>(m0 + rt) * a.hidden + slice * 64 + ch * 8) = u;
    }
  }
  stampc(11);
}

// Device-wide barrier between phases.  All CTAs are co-resident (one per SM), the counter
// only grows.  Writers: bar.sync orders every thread's writes before thread 0's gpu-scope
// fence (cumulative release); readers: acquire, then a proxy fence so the next phase's TMA
// (async proxy) observes what other CTAs stored with ordinary instructions.  `sys`: the writes
// of this phase are about to be published to peer GPUs (last step's upload) -- fence at system
// scope instead.
__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int& epoch, bool sys = false) {
  ++epoch;
  __syncthreads();
  if (threadIdx.x == 0) {
    ptx::fence_proxy_async_all();
    if (sys) __threadfence_system(); else __threadfence();
    atomicAdd(counter, 1u);
    const unsigned int target = epoch * gridDim.x;
    unsigned long long spins = 0;
    while (true) {
      unsigned int v;
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
      if (v >= target) break;
      if (++spins > (1ull << 27)) __trap();  // a lost CTA traps within seconds instead of hanging
    }
    ptx::fence_proxy_async_all();
  }
  __syncthreads();
}

// The trainer's body.  DP = false is mlp_round_kernel; DP = true (mlp_dpsgd_round_kernel) adds DP-SGD,
// every instruction of it under `if constexpr (DP)`, so the plain entries compile as before.
template <bool FP8, bool DP>
__device__ __forceinline__ void mlp_round_body(const Maps& maps, const Args& a, const TrainerDp& d) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kTileBytes);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* accum_bar = empty_bar + kStages;
  uint64_t* cbar = accum_bar + 1;      // chain barriers
  ChainBars cb{cbar, cbar + 1, cbar + 2, cbar + 3, cbar + 4, cbar + 5, cbar + 6, cbar + 7};
  float* stage_base = reinterpret_cast<float*>(smem + kTileBytes + kBarBytes);
  float* sbias = stage_base + kEpiWarps * 32 * kStgLd;
  const wg::AccTile at{sbias + kBiasFloats, kAccPitch};

  ptx::pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __shared__ int ticket;

  // The kernel body exists three times, specialised per role (producer, MMA, epilogue
  // warpgroups), each entered right after its setmaxnreg so that no value lives across the
  // register reallocation.  All copies execute the same sequence of CTA-wide and grid barriers.
  auto role_body = [&](auto role_tag) __attribute__((always_inline)) {
  constexpr int ROLE = decltype(role_tag)::value;
  if (warp == 0 && lane == 0) {
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 128);   // the MMA warpgroup's threads release a slot
    }
    ptx::mbar_init(accum_bar, 128);
    ptx::mbar_init(cb.h, 1); ptx::mbar_init(cb.w2k, 1); ptx::mbar_init(cb.w2mn, 1);
    ptx::mbar_init(cb.acc_l, 128); ptx::mbar_init(cb.acc_dh, 128);
    ptx::mbar_init(cb.dl_ready, kEpiThreads);
    ptx::mbar_init(cb.ring_free, 4 * kCluster);
    ptx::mbar_init(cb.hx, 1);
    if constexpr (DP) ptx::mbar_init(cbar + 8, kCluster * kBMx);   // DP-SGD exchange: one arrive per row and CTA
    ptx::fence_mbar_init();
  }
  __syncthreads();
  // plan 4: every CTA's barriers are initialised before any CTA of the cluster arrives on them
  if (a.chain == 4) ptx::cluster_sync();
  ptx::pdl_wait();
  if (a.pred != nullptr && *a.pred == 0) return;

  Pipe pp{0u, 0u};
  uint32_t chains = 0;        // chains processed by this CTA (parity of the once-per-chain barriers)
  bool x_all_ready = false;   // input pipeline: every chunk of this round has been converted
  unsigned int bar_epoch = 0;
  const int t = blockIdx.x;
  const int q = warp & 3, half = (warp - 4) >> 2;       // epilogue warps 4..11
  float* stg = stage_base + (warp >= 4 && warp < kProducerWarp ? warp - 4 : 0) * (32 * kStgLd);
  const int B = a.B, H = a.hidden, C = a.n_classes, D = a.in_dim;
  const int mt_b = (B + kBM - 1) / kBM;                 // M-tiles over the batch
  const int nt_h = (H + kBN - 1) / kBN;                 // N-tiles over hidden
  const int nt_d = (D + kBN - 1) / kBN;                 // N-tiles over in_dim
  const int bm_w = a.bm_w;                              // weight-gradient tile height (64 | 128)
  const int mt_hw = (H + bm_w - 1) / bm_w;              // M-tiles over hidden (dW1)
  const int kb_d = (D + 63) / 64, kb_h = (H + 63) / 64, kb_b = (B + 63) / 64, kb_c = (C + 63) / 64;
  const bool fused = a.chain == 4;
  const int bm_x = fused ? kBMx : kBM;                  // M-tile height of fwd1 and the chain
  const int mt_x = (B + bm_x - 1) / bm_x;
  const int p1_tiles = mt_x * nt_h;
  uint32_t mk = 0u;           // plan 4: relu mask the fwd1 epilogue hands to chain step E3

  auto run = [&](const Job& j) {
    if constexpr (ROLE == kRoleEpi) epilogue_tile<FP8>(j, a, q, half, lane, accum_bar, at, stg, sbias, pp);
    else if constexpr (ROLE == kRoleMma) mma_tile(j, smem, full_bar, empty_bar, accum_bar, at, pp, nullptr, &a);
    else if (warp == kProducerWarp) produce_tile(j, smem, full_bar, empty_bar, pp);
  };
  // DP-SGD: phase B's tiles add the noise of step word `word` (and on the last step fill the hook)
  auto run_dp = [&](const Job& j, uint32_t word, float* hook) {
    if constexpr (ROLE == kRoleEpi) epilogue_tile<FP8>(j, a, q, half, lane, accum_bar, at, stg, sbias, pp);
    else if constexpr (ROLE == kRoleMma)
      mma_tile<true>(j, smem, full_bar, empty_bar, accum_bar, at, pp, nullptr, &a, &d, word, hook);
    else if (warp == kProducerWarp) produce_tile(j, smem, full_bar, empty_bar, pp);
  };

  // Phase plan of one step (a.chain, a.epiopt pick the variant; all are numerically equivalent):
  //   chain 4:  [P1 fwd1 -> h on chip -> fwd2 -> xent -> dh] per M-tile cluster | B
  //   chain 3:  P1 fwd1 | [fwd2 -> xent -> dh chained per M-tile]             | B
  //   chain 0:  P1 | P2 xent | P3 dh                                          | B   (any hidden size)
  //   B = dW1 || dW2 (+ SGD/Adam in the epilogue and a bias CTA when epiopt, else a flat P5)
  auto stamp = [&](int step, int slot) {
    if (a.dbg != nullptr && blockIdx.x == 0 && threadIdx.x == kEpiT0) a.dbg[step * 32 + slot] = globaltimer_ns();
  };
  for (int step = 0; step < a.steps; ++step) {
    const int r0 = (step % a.epoch_steps) * B;   // local epoch k > 0 repeats epoch 0's batches
    const bool last = step == a.steps - 1;
    float bc1 = 1.f, bc2 = 1.f;
    if (a.adam) {
      const int tt = (a.step_base ? *a.step_base : 0) + step + 1;
      bc1 = 1.f - powf(a.beta1, static_cast<float>(tt));
      bc2 = 1.f - powf(a.beta2, static_cast<float>(tt));
    }
    const bool eo = a.epiopt != 0;
    unsigned long long* sdbg = a.dbg != nullptr ? a.dbg + step * 32 : nullptr;
    // DP-SGD: the noise's step word, and the released-gradient hook of the last step
    [[maybe_unused]] uint32_t dp_word = 0;
    [[maybe_unused]] float* dp_hook = nullptr;
    if constexpr (DP) {
      dp_word = static_cast<uint32_t>((a.step_base ? *a.step_base : 0) + step);
      if (last && d.dbg != nullptr) dp_hook = d.dbg + static_cast<long long>(a.steps) * 5 * B;
    }
    stamp(step, 0);
    // ---- P1: h = relu(x W1^T + b1)
    if (t < p1_tiles) {
      if (ROLE == kRoleProducer && a.x_ready != nullptr && warp == kProducerWarp && !x_all_ready) {
        // input pipeline: this step's rows are converted by the side-branch kernel as soon as
        // their H2D copy lands; only the TMA producer has to wait (phase B reads them later).
        // Once the LAST chunk (E - 1) is seen ready nothing is checked any more: later local epochs
        // read the same E chunks again.
        int all = 0;
        if (lane == 0) {
          const unsigned int want = __ldcg(a.round_seq) + 1u;   // bumped by k_consensus at round end
          unsigned int v;
          asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.x_ready + a.epoch_steps - 1) : "memory");
          all = static_cast<int>(v - want) >= 0 ? 1 : 0;
          unsigned long long spins = 0;
          while (!all) {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.x_ready + step % a.epoch_steps) : "memory");
            if (static_cast<int>(v - want) >= 0) break;
            if (++spins > (1ull << 28)) __trap();   // the input kernel gives up (error word) long before this
            __nanosleep(32);
          }
        }
        x_all_ready = __shfl_sync(0xffffffffu, all, 0) != 0;
        ptx::fence_proxy_async_all();   // their generic stores -> this warp's TMA (async proxy) loads
      }
      Job j{};
      j.mode = E_BIAS_RELU_BF16; j.d = a.h; j.ldd = H; j.bias = a.b1; j.M = B; j.N = H; j.bm = bm_x;
      j.dbg = sdbg; j.dbg_slot = 16;
      j.m0 = (t / nt_h) * bm_x; j.n0 = (t % nt_h) * kBN;
      j.ta = &maps.x_k; j.tb = &maps.w1_k; j.a_mn = 0; j.b_mn = 0;
      j.a_c0 = 0; j.a_c1 = r0 + j.m0; j.b_c0 = 0; j.b_c1 = j.n0; j.n_kb = kb_d;
      if (!fused) {
        run(j);
      } else {
        // plan 4 (hidden = 256: P1 tile t is chain CTA t, rank t % 4 of M-tile t / 4's cluster)
        const uint32_t par = chains & 1;
        if constexpr (ROLE == kRoleEpi) {
          if constexpr (DP) mk = fwd1_epilogue_x<FP8, true>(j, a, smem, cb, lane, accum_bar, at, sbias, pp, par, t % 4, &d);
          else mk = fwd1_epilogue_x<FP8>(j, a, smem, cb, lane, accum_bar, at, sbias, pp, par, t % 4);
        } else if constexpr (ROLE == kRoleMma) {
          mma_tile(j, smem, full_bar, empty_bar, accum_bar, at, pp, cb.ring_free);
        } else if (warp == kProducerWarp) {
          produce_tile(j, smem, full_bar, empty_bar, pp);
          // W2 lands in ring stages 2-4: wait until the MMA released the last K-block's stage (the
          // ring is drained), then load it underneath the fwd1 epilogue
          const uint32_t last = pp.it - 1;
          ptx::mbar_wait(&empty_bar[last % kStages], (last / kStages) & 1);
          chain_produce(maps, smem, cb, j.m0, t % 4, false);
        }
      }
    }
    if (!fused) {
      grid_barrier(a.barrier, bar_epoch);
      stamp(step, 1);
    }
    if (a.chain != 0) {
      // ---- chained tail of the forward/backward pass per M-tile: four CTAs per M-tile, each
      // redoes fwd2 + xent (cheap) and owns a 64-column slice of dh
      if (t < mt_x * 4) {
        const int m0 = (t / 4) * bm_x, slice = t % 4;
        const uint32_t par = chains & 1;
        if constexpr (ROLE == kRoleEpi) {
          if constexpr (DP)
            chain_epilogue<kBMx, true>(a, smem, cb, at, lane, stage_base, sbias, par, m0, r0, slice, sdbg, true, mk,
                                       &d, cbar + 8, step);
          else if (fused) chain_epilogue<kBMx>(a, smem, cb, at, lane, stage_base, sbias, par, m0, r0, slice, sdbg, true, mk);
          else chain_epilogue<kBM>(a, smem, cb, at, lane, stage_base, sbias, par, m0, r0, slice, sdbg, false, 0u);
        } else if constexpr (ROLE == kRoleMma) {
          if (fused) chain_mma<kBMx>(smem, cb, at, par, true);
          else chain_mma<kBM>(smem, cb, at, par, false);
        } else if (warp == kProducerWarp && !fused) chain_produce(maps, smem, cb, m0, slice, true);
        ++chains;
      }
      grid_barrier(a.barrier, bar_epoch);
      stamp(step, 2);
    } else {
      // ---- P2: logits -> dlogits / loss / db2
      if (t < mt_b) {
        Job j{};
        j.ta = &maps.h_k; j.tb = &maps.w2_k; j.a_mn = 0; j.b_mn = 0; j.bm = kBM;
        j.m0 = t * kBM; j.n0 = 0; j.M = B; j.N = C;
        j.a_c0 = 0; j.a_c1 = j.m0; j.b_c0 = 0; j.b_c1 = 0; j.n_kb = kb_h;
        j.mode = E_XENT; j.d = a.dlogits; j.ldd = a.ncp; j.bias = a.b2; j.colsum = a.gb2;
        j.labels = a.labels + r0; j.grad_scale = 1.f / static_cast<float>(B);
        run(j);
      }
      grid_barrier(a.barrier, bar_epoch);
      // ---- P3: dh = (dlogits W2) * relu'(h), db1
      if (t < mt_b * nt_h) {
        Job j{};
        j.ta = &maps.dl_k; j.tb = &maps.w2_mn; j.a_mn = 0; j.b_mn = 1; j.bm = kBM;
        j.m0 = (t / nt_h) * kBM; j.n0 = (t % nt_h) * kBN; j.M = B; j.N = H;
        j.a_c0 = 0; j.a_c1 = j.m0; j.b_c0 = j.n0; j.b_c1 = 0; j.n_kb = kb_c;
        j.mode = E_MASK_COLSUM_BF16; j.d = a.dh; j.ldd = H; j.aux = a.h; j.colsum = a.gb1;
        run(j);
      }
      grid_barrier(a.barrier, bar_epoch);
      stamp(step, 2);
    }
    // ---- B: dW1 = dh^T x (tiles [0, mt_hw*nt_d))  ||  dW2 = dlogits^T h (next nt_h tiles)  || biases
    if (t < mt_hw * nt_d) {
      Job j{};
      j.ta = &maps.dh_mn; j.tb = &maps.x_mn; j.a_mn = 1; j.b_mn = 1; j.bm = bm_w;
      j.m0 = (t / nt_d) * bm_w; j.n0 = (t % nt_d) * kBN; j.M = H; j.N = D;
      j.a_c0 = j.m0; j.a_c1 = 0; j.b_c0 = j.n0; j.b_c1 = r0; j.n_kb = kb_b;
      j.mode = eo ? E_OPT : E_F32; j.d = eo ? a.master + (a.gw1 - a.grad) : a.gw1; j.ldd = D;
      j.bc1 = bc1; j.bc2 = bc2; j.last = last ? 1 : 0;
      // fp8 mode: no GEMM reads W1's bf16 shadow (fwd1 takes work_dq), so only the last step
      // writes it, leaving it bf16 of the final master as in bf16 mode
      j.shadow = !FP8 || last;
      j.dbg = sdbg; j.dbg_slot = 18;
      j.q_off = a.ql.w1q; j.qsf_off = a.ql.w1sf; j.ldq = D; j.q_nkb = a.ql.kb1; j.dq_off = 0;
      if constexpr (DP) run_dp(j, dp_word, dp_hook);
      else run(j);
    } else if (t < mt_hw * nt_d + nt_h) {
      const int u = t - mt_hw * nt_d;
      Job j{};
      j.ta = &maps.dl_mn; j.tb = &maps.h_mn; j.a_mn = 1; j.b_mn = 1; j.bm = bm_w;
      j.m0 = 0; j.n0 = u * kBN; j.M = C; j.N = H;
      j.a_c0 = 0; j.a_c1 = 0; j.b_c0 = j.n0; j.b_c1 = 0; j.n_kb = kb_b;
      j.mode = eo ? E_OPT : E_F32; j.d = eo ? a.master + (a.gw2 - a.grad) : a.gw2; j.ldd = H;
      j.bc1 = bc1; j.bc2 = bc2; j.last = last ? 1 : 0;
      j.shadow = 1;   // dh's B operand (w2_mn) reads W2's shadow in both modes
      j.q_off = a.ql.w2q; j.qsf_off = a.ql.w2sf; j.ldq = H; j.q_nkb = a.ql.kb2;
      j.dq_off = static_cast<long long>(H) * D;
      if constexpr (DP) run_dp(j, dp_word, dp_hook);
      else run(j);
    } else if (eo && t == mt_hw * nt_d + nt_h) {
      // biases: their gradients were accumulated by column sums earlier in the step; consume + re-zero
      const bool up = last && a.has_fed;
      UploadDst ud{};
      if (up) ud = upload_dst<FP8>(a);
      if constexpr (DP) {
        // the noise of b1 | b2, one dp_gauss4 call per 4 consecutive flat indices (both offsets are multiples
        // of 8), parked in sbias at the workspace's column layout (b1 at i, b2 at kChainH + i)
        if (d.sigma > 0.f) {
          const int g1 = H / 4, g2 = (C + 3) / 4;
          for (int k = threadIdx.x; k < g1 + g2; k += blockDim.x) {
            const bool w1 = k < g1;
            const int col = w1 ? 4 * k : kChainH + 4 * (k - g1);
            const long long pn = (w1 ? a.gb1 + 4 * k : a.gb2 + 4 * (k - g1)) - a.grad;
            float z[4];
            dp_gauss4(d.seed, dp_word, static_cast<uint64_t>(pn >> 2), z, kDpsgdSite);
#pragma unroll
            for (int q = 0; q < 4; ++q) sbias[col + q] = z[q];
          }
        }
        __syncthreads();
      }
      for (int i = threadIdx.x; i < H + C; i += blockDim.x) {
        float* gp = i < H ? a.gb1 + i : a.gb2 + (i - H);
        float g;
        if constexpr (DP) {
          // the M-tiles' 32-row column sums of dh' | dz' in M-tile order, then the noise
          const int col = i < H ? i : kChainH + (i - H);
          const float* ws = d.bias_ws + col;
          g = 0.f;
          for (int p = 0; p < 2 * mt_x; ++p) g = so_add(g, __ldcg(ws + static_cast<long long>(p) * kDpWsLd));
          if (d.sigma > 0.f) g = so_add(g, so_mul(d.sigma, sbias[col]));
          if (dp_hook != nullptr) dp_hook[gp - a.grad] = g;
        } else {
          g = __ldcg(gp);
          *gp = 0.f;
        }
        float w[4];
        const long long pi = gp - a.grad;
        opt_apply(a, pi, 1, &g, bc1, bc2, w);
        if (up) {
          float wu = w[0];
          if (ud.global != nullptr) { const float g0 = __ldcg(ud.global + pi); wu = g0 - ud.byz_scale * (wu - g0); }
          ud.master[pi] = wu;
          ud.shadow[pi] = __float2bfloat16(wu);
          if (FP8) *reinterpret_cast<float*>(ud.blob + (i < H ? a.ql.b1 + 4 * i : a.ql.b2 + 4 * (i - H))) = wu;
        }
      }
    }
    stamp(step, 3);
    grid_barrier(a.barrier, bar_epoch, last && a.has_fed);
    stamp(step, 4);
    if (eo) continue;   // the optimizer ran in the epilogues
    // ---- P5: optimizer over the flat buffer (all threads of all CTAs)
    {
      const long long nv = a.n_params / 4;
      const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
      for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv; i += stride) {
        const float4 g4 = __ldcg(reinterpret_cast<const float4*>(a.grad) + i);
        const float g[4] = {g4.x, g4.y, g4.z, g4.w};
        float w[4];
        opt_apply(a, 4 * i, 4, g, bc1, bc2, w);
        reinterpret_cast<float4*>(a.grad)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    grid_barrier(a.barrier, bar_epoch);
    stamp(step, 5);
  }

  // ---- UploadLocalUpdate, second half: every CTA's upload stores were fenced at system scope
  // before the last barrier; CTA 0 pushes the meta record into every replica's ledger page and
  // raises FLAG_TRAINED on every peer (C:246-253).
  if (a.has_fed && a.epiopt && blockIdx.x == 0) {
    char* me = a.f.peers.base[a.f.rank];
    const RoundState* st = heap_at<const RoundState>(me, a.f.lay.state_off);
    RoundPlan* plan = heap_at<RoundPlan>(me, a.f.lay.plan_off);
    const uint32_t epoch = st->epoch;
    const uint32_t par = epoch & 1u;
    if (threadIdx.x == 0) atomicMax(&plan->t_stamp[STAMP_UPLOAD_BEGIN], globaltimer_ns());
    // first-K-wins admission (C:239-244): one ticket per trainer and round from the counter on
    // rank 0's page; a ticket beyond NEEDED_UPDATE_COUNT publishes nothing (update dropped)
    const bool fk = admit::first_k(st);
    if (threadIdx.x == 0) {
      admit::straggle(a.straggle_us);
      int tk = fk ? admit::take_ticket(&admit::page(a.f.peers.base[0], a.f.lay, par)->ticket, epoch) : 0;
      if (fk && tk >= static_cast<int>(st->n_needed)) tk = -1;
      ticket = tk;
    }
    __syncthreads();
    if (ticket >= 0 && threadIdx.x < a.f.n_ranks) {
      const int r = threadIdx.x;
      UploadMeta* meta = heap_at<UploadMeta>(a.f.peers.base[r], a.f.lay.meta_off) + par * kMaxRanks + a.f.rank;
      UploadMeta m;
      m.n_samples = static_cast<uint32_t>(a.n_samples);
      m.avg_cost = __ldcg(a.loss_sum) / static_cast<float>(a.n_loss_terms > 0 ? a.n_loss_terms : 1);
      *meta = m;
      __threadfence_system();
      if (fk)
        ptx::st_release_sys(&admit::page(a.f.peers.base[r], a.f.lay, par)->slot[ticket],
                            ((epoch + 1u) << 8) | static_cast<uint32_t>(a.f.rank));
      ptx::st_release_sys(heap_at<uint32_t>(a.f.peers.base[r], a.f.lay.flags_off) + FLAG_TRAINED + a.f.rank,
                          epoch + 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) atomicMax(&plan->t_stamp[STAMP_UPLOAD_END], globaltimer_ns());
  }
  };   // role_body

  if (warp < 4) {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kMmaRegs));
    role_body(std::integral_constant<int, kRoleMma>{});
  } else if (warp >= kProducerWarp) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    role_body(std::integral_constant<int, kRoleProducer>{});
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kEpiRegs));
    role_body(std::integral_constant<int, kRoleEpi>{});
  }
}

template <bool FP8>
__global__ void __launch_bounds__(kThreads, 1)
mlp_round_kernel(const __grid_constant__ Maps maps, const Args a) {
  mlp_round_body<FP8, false>(maps, a, TrainerDp{});
}

// DP-SGD entry of the trainer (plan 4, optimizer in the epilogue): its own kernel, so the plain one stays as it is
template <bool FP8>
__global__ void __launch_bounds__(kThreads, 1)
mlp_dpsgd_round_kernel(const __grid_constant__ Maps maps, const Args a, const __grid_constant__ TrainerDp d) {
  mlp_round_body<FP8, true>(maps, a, d);
}

}  // namespace

Mx8MlpLayout mx8_mlp_layout(int in_dim, int hidden) {
  Mx8MlpLayout l;
  l.kb1 = (in_dim + 127) / 128;
  l.kb2 = (hidden + 127) / 128;
  const int rb1 = (hidden + 127) / 128;
  int cur = 0;
  auto take = [&](int bytes) { const int o = cur; cur += (bytes + 127) / 128 * 128; return o; };
  l.w1q = take(hidden * in_dim);
  l.w1sf = take(rb1 * l.kb1 * epi::kSfChunk);
  l.w2q = take(64 * hidden);
  l.w2sf = take(l.kb2 * epi::kSfChunk);
  l.b1 = take(hidden * 4);
  l.b2 = take(64 * 4);
  l.total = cur;
  return l;
}

Mx8Unpack mx8_unpack_args(int in_dim, int hidden, int n_classes, long long w1_off, long long w2_off) {
  const Mx8MlpLayout l = mx8_mlp_layout(in_dim, hidden);
  Mx8Unpack u;
  u.in_dim = in_dim; u.hidden = hidden; u.n_classes = n_classes; u.w1_off = w1_off; u.w2_off = w2_off;
  u.w1q = l.w1q; u.w1sf = l.w1sf; u.w2q = l.w2q; u.w2sf = l.w2sf; u.b1 = l.b1; u.kb1 = l.kb1; u.kb2 = l.kb2;
  return u;
}

cudaError_t mlp_round_plan(const MlpPlanRequest& q, MlpRoundPlan* out) {
  if (q.hidden % 8 || q.in_dim % 8 || q.batch % 8 || q.ncp % 8 || q.n_classes > 64) return cudaErrorInvalidValue;
  const int mt_b = (q.batch + kBM - 1) / kBM, nt_h = (q.hidden + kBN - 1) / kBN;
  const int nt_d = (q.in_dim + kBN - 1) / kBN;
  // phase plan: q.plan / q.epiopt when >= 0, else BFLC_MLP_CHAIN = 0 | 3 | 4 and BFLC_MLP_EPIOPT = 0 | 1
  // (see the kernel), else the defaults
  static const int chain_env0 = [] { const char* e = std::getenv("BFLC_MLP_CHAIN"); return e ? std::atoi(e) : kDefaultPlan; }();
  static const bool epiopt_env0 = [] { const char* e = std::getenv("BFLC_MLP_EPIOPT"); return !(e && e[0] == '0'); }();
  const int chain_env = q.plan >= 0 ? q.plan : chain_env0;
  const bool epiopt = q.epiopt >= 0 ? q.epiopt != 0 : epiopt_env0;
  // the chain's fwd2 / dh tiles are 64 classes wide: ncp == 64 (57..64 classes)
  const bool chain_ok = q.hidden == kChainH && q.ncp == 64 && q.n_classes <= 64;
  int chain = (!chain_ok || chain_env == 0) ? 0 : chain_env == 4 ? 4 : 3;
  const bool fp8 = q.fp8, dp = q.dpsgd;
  if (fp8 && (chain == 0 || !epiopt || q.batch % 128 || q.in_dim % 16)) return cudaErrorNotSupported;
  // DP-SGD: plan 4 (the default) with the optimizer in the epilogue only
  if (dp && (chain != 4 || !epiopt)) return cudaErrorNotSupported;
  // weight-gradient tiles: 64 rows (one m64 wgmma) spread the optimizer epilogue over twice the CTAs;
  // BFLC_MLP_BMW=128 keeps the 128-row tiles
  static const int bmw_env = [] { const char* e = std::getenv("BFLC_MLP_BMW"); return e && std::atoi(e) == 128 ? 128 : 64; }();
  int bm_w = bmw_env;
  int mt_hw = (q.hidden + bm_w - 1) / bm_w;
  // every CTA must be resident at once (grid barriers): at most one per SM of this device
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return cudaErrorInvalidDevice;
  if (mt_hw * nt_d + nt_h + 1 > sms) { bm_w = 128; mt_hw = (q.hidden + 127) / 128; }
  // CTAs of a plan: P1 tiles, phase-B tiles (+ the bias CTA), chain CTAs.  Plan 4 runs fwd1 and the
  // chain on 64-row M-tiles, plans 0 and 3 on 128-row ones.
  auto need = [&](int ch) {
    const int mt_x = ch == 4 ? (q.batch + kBMx - 1) / kBMx : mt_b;
    return std::max({mt_x * nt_h, mt_hw * nt_d + nt_h + 1, ch != 0 ? mt_x * 4 : 0, kGrid});
  };
  int grid = need(chain);
  if (chain != 4 && grid > sms) return cudaErrorInvalidValue;

  // a FedProx launch also stages the anchor of its weight-gradient tile in shared memory
  const int smem = q.prox ? kSmemProx : kSmemTotal;
  static bool configured[2] = {false, false};
  if (!configured[fp8 ? 1 : 0]) {
    const cudaError_t ea =
        fp8 ? cudaFuncSetAttribute(mlp_round_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemProx)
            : cudaFuncSetAttribute(mlp_round_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemProx);
    if (ea != cudaSuccess) return ea;
    configured[fp8 ? 1 : 0] = true;
  }
  static bool configured_dp[2] = {false, false};
  if (dp && !configured_dp[fp8 ? 1 : 0]) {
    const cudaError_t ea =
        fp8 ? cudaFuncSetAttribute(mlp_dpsgd_round_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemProx)
            : cudaFuncSetAttribute(mlp_dpsgd_round_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemProx);
    if (ea != cudaSuccess) return ea;
    configured_dp[fp8 ? 1 : 0] = true;
  }
  int mc_out = 0;
  if (chain == 4) {
    // Plan 4 launches clusters of 4 (the grid rounded up to whole clusters), and the grid barriers
    // still need every CTA resident at once: where the device cannot hold that many clusters, plan 3.
    static int max_clusters[2][2][2] = {{{-1, -1}, {-1, -1}}, {{-1, -1}, {-1, -1}}};
    int& mc = max_clusters[dp ? 1 : 0][fp8 ? 1 : 0][q.prox ? 1 : 0];
    const int grid4 = (grid + kCluster - 1) / kCluster * kCluster;
    if (mc < 0) {
      cudaLaunchConfig_t cfg{};
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = kCluster; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
      cfg.gridDim = dim3(grid4);
      cfg.blockDim = dim3(kThreads);
      cfg.dynamicSmemBytes = smem;
      cfg.attrs = attr;
      cfg.numAttrs = 1;
      int n = 0;
      const cudaError_t eo =
          dp ? (fp8 ? cudaOccupancyMaxActiveClusters(&n, mlp_dpsgd_round_kernel<true>, &cfg)
                    : cudaOccupancyMaxActiveClusters(&n, mlp_dpsgd_round_kernel<false>, &cfg))
             : (fp8 ? cudaOccupancyMaxActiveClusters(&n, mlp_round_kernel<true>, &cfg)
                    : cudaOccupancyMaxActiveClusters(&n, mlp_round_kernel<false>, &cfg));
      if (eo != cudaSuccess) { (void)cudaGetLastError(); n = 0; }
      mc = n;
    }
    mc_out = mc;
    if (grid4 <= sms && mc * kCluster >= grid4) {
      grid = grid4;
    } else {
      if (dp) {   // DP-SGD has no plan-3 form
        out->plan = 4; out->epiopt = epiopt; out->grid = grid4; out->bm_w = bm_w; out->max_clusters = mc;
        return cudaErrorNotSupported;
      }
      chain = 3;
      grid = need(3);
      if (grid > sms) return cudaErrorInvalidValue;
    }
  }
  out->plan = chain; out->epiopt = epiopt; out->grid = grid; out->bm_w = bm_w; out->max_clusters = mc_out;
  return cudaSuccess;
}

cudaError_t mlp_round_sm100(const MlpRoundArgs& r, cudaStream_t stream) {
  bind_context_once();
  // the rows of one local epoch: whole batches, at most one per step
  if (r.steps < 1 || r.epoch_rows < r.batch || r.epoch_rows % r.batch ||
      r.epoch_rows / r.batch > r.steps)
    return cudaErrorInvalidValue;
  if (r.n_params % 4) return cudaErrorInvalidValue;
  const bool fp8 = r.fp8;
  if (fp8 && (!r.x_dq || !r.work_q || !r.work_dq || !r.h_dq)) return cudaErrorNotSupported;
  if (r.prox_anchor != nullptr && (reinterpret_cast<uintptr_t>(r.prox_anchor) % 16 || !(r.prox_mu > 0.f)))
    return cudaErrorInvalidValue;   // the anchor is read as float4
  const MlpDpsgdArgs* dp = r.dpsgd;
  if (dp != nullptr &&
      (!(std::isfinite(dp->clip) && dp->clip > 0.f) || !(std::isfinite(dp->sigma) && dp->sigma >= 0.f) ||
       dp->dropped == nullptr || dp->bias_ws == nullptr || r.x == nullptr))
    return cudaErrorInvalidValue;
  MlpPlanRequest q;
  q.batch = r.batch; q.in_dim = r.in_dim; q.hidden = r.hidden; q.n_classes = r.n_classes; q.ncp = r.ncp;
  q.plan = r.plan; q.epiopt = r.epiopt; q.fp8 = fp8; q.dpsgd = dp != nullptr; q.prox = r.prox_anchor != nullptr;
  MlpRoundPlan pl;
  const cudaError_t ep = mlp_round_plan(q, &pl);
  if (ep != cudaSuccess) return ep;
  if (r.fed != nullptr && !pl.epiopt) return cudaErrorNotSupported;
  const int chain = pl.plan, grid = pl.grid, bm_w = pl.bm_w;
  const bool epiopt = pl.epiopt;
  const int smem = q.prox ? kSmemProx : kSmemTotal;

  Maps m;
  std::memset(&m, 0, sizeof(m));
  const long long rows_x = r.epoch_rows;
  auto mk = [&](CUtensorMap* out, const void* ptr, long long ld, bool mn, int rows_extent, int K,
                int rows_tile, DType dt = DType::BF16) {
    GemmOperand op{ptr, ld, 0, mn};
    return gemm_make_operand_map(out, op, dt, rows_extent, K, 1, rows_tile);
  };
  cudaError_t e;
  // K-major: (rows_extent = M|N, K);  MN-major: memory [K][M|N].  The K-major A operands (x, h,
  // dlogits) are 64-row boxes: one per m64 half of a tile (produce_tile, chain_produce).
  // the forward operands: bf16 shadows, or in fp8 mode the exactly dequantised MXFP8 copies
  const void* fx = fp8 ? r.x_dq : r.x;
  const void* fw1 = fp8 ? static_cast<const void*>(r.work_dq) : r.w1_shadow;
  const void* fh = fp8 ? r.h_dq : r.h;
  const void* fw2 = fp8 ? static_cast<const void*>(r.work_dq + static_cast<long long>(r.hidden) * r.in_dim)
                        : r.w2_shadow;
  if ((e = mk(&m.x_k, fx, r.in_dim, false, (int)rows_x, r.in_dim, 64)) != cudaSuccess) return e;
  if ((e = mk(&m.w1_k, fw1, r.in_dim, false, r.hidden, r.in_dim, kBN)) != cudaSuccess) return e;
  if ((e = mk(&m.h_k, fh, r.hidden, false, r.batch, r.hidden, 64)) != cudaSuccess) return e;
  if ((e = mk(&m.w2_k, fw2, r.hidden, false, r.n_classes, r.hidden, kBN)) != cudaSuccess) return e;
  if ((e = mk(&m.dl_mn, r.dlogits, r.ncp, true, r.n_classes, r.batch, kBM)) != cudaSuccess) return e;
  if ((e = mk(&m.h_mn, r.h, r.hidden, true, r.hidden, r.batch, kBN)) != cudaSuccess) return e;
  if ((e = mk(&m.dl_k, r.dlogits, r.ncp, false, r.batch, r.n_classes, 64)) != cudaSuccess) return e;
  if ((e = mk(&m.w2_mn, r.w2_shadow, r.hidden, true, r.hidden, r.n_classes, kBN)) != cudaSuccess) return e;
  if ((e = mk(&m.dh_mn, r.dh, r.hidden, true, r.hidden, r.batch, kBM)) != cudaSuccess) return e;
  if ((e = mk(&m.x_mn, r.x, r.in_dim, true, r.in_dim, (int)rows_x, kBN)) != cudaSuccess) return e;
  const Mx8MlpLayout ql = mx8_mlp_layout(r.in_dim, r.hidden);

  Args a{};
  a.B = r.batch; a.steps = r.steps; a.epoch_steps = r.epoch_rows / r.batch; a.in_dim = r.in_dim; a.hidden = r.hidden;
  a.n_classes = r.n_classes; a.ncp = r.ncp; a.n_params = r.n_params;
  a.chain = chain; a.epiopt = epiopt ? 1 : 0; a.dbg = r.dbg;
  a.x_ready = r.x_ready; a.round_seq = r.round_seq;
  a.pred = r.pred ? r.pred : current_predicate();
  a.barrier = r.barrier;
  a.master = r.master; a.b1 = r.b1; a.b2 = r.b2;
  a.grad = r.grad; a.gw1 = r.gw1; a.gb1 = r.gb1; a.gw2 = r.gw2; a.gb2 = r.gb2;
  a.shadow = reinterpret_cast<__nv_bfloat16*>(r.shadow);
  a.adam_m = r.adam_m; a.adam_v = r.adam_v; a.adam = r.adam ? 1 : 0;
  a.lr = r.lr; a.beta1 = r.beta1; a.beta2 = r.beta2; a.eps = r.eps; a.step_base = r.step_base;
  a.h = reinterpret_cast<__nv_bfloat16*>(r.h);
  a.dlogits = reinterpret_cast<__nv_bfloat16*>(r.dlogits);
  a.dh = reinterpret_cast<__nv_bfloat16*>(r.dh);
  a.labels = r.labels; a.loss_sum = r.loss_sum; a.correct = r.correct;
  a.work_q = r.work_q; a.work_dq = reinterpret_cast<__nv_bfloat16*>(r.work_dq);
  a.h_dq = reinterpret_cast<__nv_bfloat16*>(r.h_dq); a.ql = ql; a.bm_w = bm_w;
  a.has_fed = r.fed != nullptr ? 1 : 0;
  if (r.fed != nullptr) a.f = *r.fed;
  a.upq_off[0] = r.upq_off[0]; a.upq_off[1] = r.upq_off[1];
  a.n_samples = r.n_samples; a.n_loss_terms = r.n_loss_terms; a.byz_mode = r.byz_mode; a.byz_scale = r.byz_scale;
  a.straggle_us = r.straggle_us;
  a.prox_anchor = r.prox_anchor; a.prox_mu = r.prox_mu;

  note_launch();
  const unsigned cluster = chain == 4 ? kCluster : 1u;
  if (dp != nullptr) {
    TrainerDp d{};
    d.clip = dp->clip; d.sigma = dp->sigma; d.bsz = static_cast<float>(r.batch); d.seed = dp->seed;
    d.x = reinterpret_cast<const __nv_bfloat16*>(r.x);
    d.dropped = dp->dropped; d.bias_ws = dp->bias_ws; d.dbg = dp->dbg;
    if (fp8) return launch_pdl_cluster(cluster, mlp_dpsgd_round_kernel<true>, dim3(grid), dim3(kThreads), smem, stream, m, a, d);
    return launch_pdl_cluster(cluster, mlp_dpsgd_round_kernel<false>, dim3(grid), dim3(kThreads), smem, stream, m, a, d);
  }
  if (fp8) return launch_pdl_cluster(cluster, mlp_round_kernel<true>, dim3(grid), dim3(kThreads), smem, stream, m, a);
  return launch_pdl_cluster(cluster, mlp_round_kernel<false>, dim3(grid), dim3(kThreads), smem, stream, m, a);
}

}  // namespace bflc
