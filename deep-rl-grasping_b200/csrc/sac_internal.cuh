// Internal declarations shared by sac.cu (handle, step orchestration, C ABI) and engine_v2.cu (TMA-fed wgmma engine).
#pragma once
#include <cuda_runtime.h>

#include <deque>
#include <map>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/b200grasp.h"
#include "cg.cuh"
#include "common.cuh"
#include "enc_stage.cuh"
#include "host.cuh"
#include "metrics_log.cuh"
#include "obsnorm.cuh"
#include "per.cuh"

namespace b2g {
struct Tensor {
  std::string name;
  int ndim;
  int64_t shape[4];
  int64_t numel;
  int64_t off;    // float offset inside P
  int group;      // 0 pi, 1 values, 2 ent, 3 target
};


// ---- engine v2 (cg.cu): BF16 plane tensors, tensor maps and problem groups of the TMA-fed path
// conv1 reads the normalised image space-to-depth: S[sample][Y 16][X 16][b 4][c 4][ci < Cp] holds pixel (4Y + b, 4X + c), so the
// 8x8 stride-4 convolution is a 2x2 stride-1 one over S.  Cp = 1 for one channel, else 4 (zero pad channels): conv1's operand
// rows are two neighbouring blocks (64 bytes) or one block (128 bytes), swizzle spans that TMA and wgmma share.
__host__ __device__ constexpr int s2d_channels(int Ci) { return Ci == 1 ? 1 : 4; }
// conv1's K index (window (a, a') = (ky / 4, kx / 4), then (b, c, ci) = (ky % 4, kx % 4, ci)) of HWIO weight row (ky * 8 + kx) * Ci + ci
__host__ __device__ inline int conv1_krow(int r, int Ci) {
  const int ci = r % Ci, kx = (r / Ci) % 8, ky = r / (8 * Ci);
  return ((((ky >> 2) * 2 + (kx >> 2)) * 4 + (ky & 3)) * 4 + (kx & 3)) * s2d_channels(Ci) + ci;
}
struct V2State {
  bool on = false;               // the step runs on this engine (CNN policy, 64 x 64 input, bf16x3)
  int KF = 576;                 // feature-row width of the F planes (513 features + actions, zero padded to 9 x 64)
  // activations: [which / net][plane]
  uint16_t* S[2][3]{};           // the normalised image space-to-depth: [B][16][16][4][4][Cp]  (0 = obs, 1 = next_obs)
  uint16_t* H1[3][3]{};          // [B*225][32]
  uint16_t* H2[3][3]{};          // [B*36][64]
  uint16_t* H3[3][3]{};          // [B][1024]
  uint16_t* F[3][3]{};           // [B][KF]
  // gradient maps, 2 planes
  uint16_t* dz0pi[2]{};          // [B][H]
  uint16_t* dz0v[2]{};           // [B][3H]
  uint16_t* dZ4[2][2]{};         // [net][plane] [B][512]
  uint16_t* dZ3[2][2]{};         // [B*16][64]
  uint16_t* dZ2[2][2]{};         // [B*36][64]
  uint16_t* dZ1[2]{};            // [plane] [B*225][2 nets][32]
  // weights as planes (refreshed every step by planes2_kernel)
  uint16_t* W1T[2][3]{};         // [0]: obs [64 = pi|vf][64*Cp], [1]: target [32][64*Cp]; K in conv1_krow order (pad rows zero)
  uint16_t* W2T[3][3]{};         // [net][plane] [64][512]
  uint16_t* W3T[3][3]{};         // [64][576]
  uint16_t* WfT[3][3]{};         // [512][1024]
  uint16_t* K0T[3][3]{};         // [0] pi [H][KF], [1] values vf|q1|q2 [3H][KF], [2] target vf [H][KF]
  uint16_t* W2n[2][2]{};         // natural [512][64] (dgrad B operand), nets pi / values, 2 planes
  uint16_t* W3n[2][2]{};         // [576][64]
  uint16_t* Wfn[2][2]{};         // [1024][512]
  uint16_t* K0n[2][2]{};         // [0] pi [513 -> 576 rows][H], [1] values packed [576 rows][3H]
  float* z0v = nullptr;          // fc0 pre-activations of vf|q1|q2: [B][3H]
  void* plane_jobs = nullptr; int n_plane_jobs = 0, plane_ctas = 0;
  int plane_ctas_fwd = 0;        // CTAs [0, plane_ctas_fwd) write the forward layouts (W1T .. K0T), the rest W2n .. K0n
  const int* plane_cta_job = nullptr;  // job index of every CTA of the planes launches
  int sm_reserve = 0;           // SMs left to a collective that runs concurrently with the persistent GEMM grids
  std::vector<CUtensorMap> maps; // host copy
  std::vector<char> map_whole;   // per map: the box spans every plane
  std::vector<int> map_box_bytes;
  CUtensorMap* d_maps = nullptr;
  std::vector<CgGroup> fwd, bwd_groups;   // per-layer problem groups: the parts fuse_groups concatenates
  // fused launches: the layer groups above concatenated into one persistent launch each, chained by arrival counters
  std::vector<CgGroup> fwd_fused, bwd_fused;
  int split_fc1 = 3;             // K-splits of the cnn_fc1 forward tiles (1 = none)
  int split_fc1_dgrad = 1;       // K-splits of the cnn_fc1 dgrad tiles (B2G_SPLIT_FC1_DGRAD; opt-in)
  int* dep_ctr = nullptr; int n_dep_ctr = 0;
  std::vector<int*> tabs;
  int dbg = 0;
};

}  // namespace b2g

struct b2g_sac;
namespace b2g {
int v2_alloc(b2g_sac* h);    // plane tensors (before the v1 groups are built: policy inference writes planes 0 / 1 of the activations)
int v2_create(b2g_sac* h);   // tensor maps + problem groups
int v2_planes(b2g_sac* h, bool backward, cudaStream_t s);   // the forward-layout or the backward-layout weight planes
int v2_gather(b2g_sac* h, const GatherArgs& ga, cudaStream_t s);
int v2_launch(b2g_sac* h, const CgGroup& g, cudaStream_t s);
// sac.cu hooks of the observe path (obsnorm.cu)
// policy forward on `chunk` <= batch compact rows at `rows` (device), enqueued on h->stream; the actions land in h->pi_out
int sac_act_rows(b2g_sac* h, const float* rows, int chunk, int deterministic);
}  // namespace b2g

using namespace b2g;   // (internal header: only library translation units include it)

struct b2g_sac {
  b2g_sac_cfg cfg{};
  bool cnn = false;
  int num_sms = 132;
  int B = 0, A = 0, H = 0, E = 0, Cimg = 0, feat_dim = 0, FS = 0;
  int Hi = 0, Wi = 0, H1 = 0, W1 = 0, H2 = 0, W2 = 0, H3 = 0, W3 = 0;
  std::vector<Tensor> tensors;
  std::map<std::string, int> tindex;
  int64_t n_pi = 0, n_values = 0, n_ent = 0, n_target = 0, n_train = 0, n_all = 0;
  float *P = nullptr, *Mo = nullptr, *Vo = nullptr, *G = nullptr;   // G has MET_COUNT extra floats (metrics ride the all-reduce)
  float* metrics = nullptr;
  cudaStream_t stream = nullptr;
  std::vector<void*> allocs;
  // Raw (un-normalised) observations travel as compact rows of Ec floats.  MLP policy: Ec = E.  CNN policy: COMPACT rows
  // (replay.cu), Ec = H*W*Cimg + 4: the image planes, the ONE actuator value the policy reads (pixel [0,0] of the last plane;
  // augmented_nature_cnn never reads the rest of it, custom_obs_policy.py:28-30; zero under B2G_CNN_NATURE) and 3 pad floats.  The explicit batch
  // (s_obs / s_next) and the pipelined staging (ps_obs / ps_next) hold such rows.
  int Ec = 0;
  // Replay: a ring of cap transition slots {obs frame, next_obs frame, act, rew, done} over a pool of frames, one compact row
  // each (per.cuh)
  TransitionReplay replay;
  FrameFmt row_fmt{};                // format of an fp32 compact row (explicit batch, staging)
  uint32_t u8_mask = 0;
  float* obs_stage = nullptr;        // CNN: caller observations in the full layout [stage_rows][E] on their way to compact rows
  int stage_rows = 0;
  // normalisation, in the ring layout (pads: mean 0, istd 1)
  double *d_mean = nullptr, *d_istd = nullptr, *d_normc = nullptr;   // normc: ret_istd, clip_obs, clip_rew, norm_obs, norm_rew
  double ret_istd = 1.0, clip_obs = 10.0, clip_rew = 10.0;
  int norm_obs = 0, norm_rew = 0;
  // batch buffers
  float *x_obs = nullptr, *x_next = nullptr;
  float *h1[3]{}, *h2[3]{}, *h3[3]{}, *F[3]{};
  float *dZ4[2]{}, *dZ3p[2]{}, *dZ2p[2]{}, *dZ1[2]{};   // round-1 backward only
  float *z0[5]{}, *a0[4]{}, *dz1[4]{}, *dz0_pi = nullptr, *dz0_v3 = nullptr;
  // BF16 hi/lo planes ([..][0] = hi, [..][1] = lo) of the tensors that feed forward / dgrad / wgrad contractions
  bool use_planes = false;
  uint16_t *xp[2][2]{}, *h1p[3][2]{}, *h2p[3][2]{}, *h3p[3][2]{};
  uint16_t *dZ4p[2][2]{}, *dZ3pp[2][2]{}, *dZ2pp[2][2]{}, *dZ1p[2][2]{};   // round-1 backward only
  ColsumJob* d_colsum = nullptr;
  int n_colsum = 0, colsum_ctas = 0;
  uint16_t* wp[3][4][4]{};          // [net][cnn1,cnn2,cnn3,fc1][hi, lo, hiT, loT]
  PlaneJob* d_jobs = nullptr;
  int n_jobs = 0, job_tiles = 0;
  bool planes_dirty = true;
  std::map<const int*, std::vector<int>> host_tabs;   // host copies of the offset tables (contract checks at build time)
  float *per_sample = nullptr, *pi_out = nullptr, *eps = nullptr, *rew_n = nullptr, *done_n = nullptr;
  int* indices = nullptr;
  float *s_obs = nullptr, *s_next = nullptr, *s_act = nullptr, *s_rew = nullptr, *s_done = nullptr;  // staged explicit batch
  // pipelined host-batch path: the big obs / next_obs copies ping-pong on a copy stream
  float *ps_obs[2]{}, *ps_next[2]{};
  // host-pipelined steps, compact transfer: the constant actuator plane never crosses PCIe (b2g_sac_step_host_pipelined)
  float *hc_obs[2]{}, *hc_next[2]{};   // pinned host staging, compact rows [B][Ec]
  cudaGraphExec_t pipe_graph[2]{};     // the step on staging slot j, captured once (b2g_sac_step_host_pipelined)
  int host_threads = 16;
  cudaStream_t cstream = nullptr;
  cudaEvent_t ev_h2d[2]{}, ev_consumed[2]{}, ev_met[2]{};
  float* pm_met[2]{};            // pinned: MET_COUNT floats + [log_alpha, grad log_alpha]
  long long* pm_cnt[2]{};        // pinned counters
  long long pipe_k = 0;
  bool pipe_pending = false;
  MetricsLog mlog;               // per-step metrics ring (b2g_sac_metrics_log); off: the step has no append node
  cudaEvent_t record_after_gather = nullptr;
  long long* counters = nullptr;
  double* step_consts = nullptr;
  float* d_lr = nullptr;
  float cur_lr = -1.f;
  // launches
  std::vector<GemmGroup> fwd_groups, bwd_groups, act_groups;
  cudaGraphExec_t graph_exec = nullptr;
  bool use_graph = true;
  void* nccl_comm = nullptr;
  void* nccl_comm2 = nullptr;          // second communicator: early all-reduce on the side stream
  // peer-memory data parallelism (b2g_sac_dp_export / _connect): every rank maps the others' parameter arena, gradient buffer and
  // exchange block through CUDA IPC; the optimiser kernel then IS the collective (optim.cu: dp_optim_kernel)
  // host-pipelined steps: copy / kernel schedule picked by timing both (b2g_sac_step_host_pipelined)
  bool pipe_serial = false; int pipe_tune = 0; double pipe_t0 = 0, pipe_period[2] = {0, 0};
  bool dp_p2p = false;
  int* dp_x = nullptr;                 // exchange block: int flags[2][8], float part[8][2]
  int* dp_sync = nullptr;              // local CTA counter + norm accumulators
  float* dp_recv = nullptr;            // receive arena: [src rank][my slice] gradient copies pushed by the other ranks
  float* dp_P[8]{}; float* dp_G[8]{}; int* dp_X[8]{};     // every rank's parameter arena, receive arena, exchange block (own = local)
  std::vector<void*> dp_opened;        // cudaIpcOpenMemHandle results
  int dp_skip[2][2]{};                 // float4 ranges of the gradient arena pushed by the cnn_fc1 wgrad epilogues
  cudaStream_t side = nullptr;
  cudaStream_t aux = nullptr;              // leaf work off the critical chain (zeroing, weight planes, leaf wgrads, bias sums)
  cudaStream_t aux2 = nullptr;             // the second leaf branch under the gather (bookkeeping kernel, gradient zeroing)
  cudaEvent_t ev_aux[9]{};
  bool fork_leaves = false;
  ColIds col_ids;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  bool overlap_ar = false;             // engine v2, N > 1: early all-reduce on the side stream (B2G_AR_OVERLAP=0 disables)
  int ar_sms = 8;
  ColsumJob* d_colsum_early = nullptr;
  int n_colsum_early = 0, colsum_early_ctas = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  float last_ms = 0.f;
  int launches = 0;
  std::vector<std::string> prof_names;
  float* h_met = nullptr;        // pinned: MET_COUNT floats + [log_alpha, grad log_alpha]
  long long* h_cnt = nullptr;    // pinned counters

  b2g::V2State v2;
  bool broken = false;               // a training-state load failed after it began writing: only destroy / load are accepted
  double* hp_stats[2]{};             // pinned staging of set_norm_stats (asynchronous upload, no stream sync)
  cudaEvent_t ev_stats[2]{};
  int stats_k = 0;

  // Device-resident VecNormalize observation statistics (created by b2g_obs_rms_set), their upload counts and the observation
  // encoder of b2g_sac_set_obs_encoder (MLP policy only: observe_* take raw rows and encode them into ob_full)
  ObsRms rms;
  // b2g_sac_observe_act / _add staging (allocated on first use): the frames of one call in the caller's layout, the current
  // observation of env i as a compact row, and the replay frame that already holds it (-1: none yet).
  float* ob_full[2]{};               // [stage_rows][E]: 0 = obs / next_obs, 1 = reset_obs
  float* ob_rows[2]{};               // compact rows [stage_rows + B][Ec] (the actor's gather reads B rows from any chunk start):
  int ob_k = 0;                      // ob_rows[ob_k] = current observation of env i; the other takes the next call's next_obs
  float *ob_act = nullptr, *ob_rew = nullptr, *ob_done = nullptr;
  std::vector<int64_t> ob_fid;
  int ob_n = 0;

  // CNN extractor (b2g_sac_net_cfg): B2G_CNN_AUGMENTED reads Cimg = obs_c - 1 planes plus the direct feature at column 512 of
  // the feature rows; B2G_CNN_NATURE reads Cimg = obs_c planes and has no direct feature.  Cobs = channels of a caller
  // observation.  cnn_scope: the extractor's layer scopes conv1, conv2, conv3, fc1 (sac.cu).
  int extractor = 0, Cobs = 0;
  const char* const* cnn_scope = nullptr;
  bool direct_feature() const { return cnn && extractor == B2G_CNN_AUGMENTED; }
  std::string cnn_t(const std::string& net, int layer, const char* wb) const { return net + "/" + cnn_scope[layer] + "/" + wb; }
  // scope of a head MLP's second layer: nature_cnn opens 'fc1' in model/pi before mlp() creates its dense layers there, so TF1
  // names the actor's second layer fc1_1 (INTEGRATION.md, "nature_cnn tensor names")
  std::string fc1(const std::string& head) const {
    return head + (cnn && extractor == B2G_CNN_NATURE && head == "model/pi" ? "/fc1_1" : "/fc1");
  }

  float* p(const std::string& n) { return P + tensors[tindex.at(n)].off; }
  float* g(const std::string& n) { return G + tensors[tindex.at(n)].off; }
};

