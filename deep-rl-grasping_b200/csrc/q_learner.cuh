// The replay Q-learner that the BDQ (bdq.cu) and DQN (dqn.cu) handles share (q_learner.cu): the parameter and Adam arenas, the
// transition replay, the normalisation table the gather reads, the batch and explicit-batch buffers, the device counters and
// the metrics ring, and what both handles do with them: set-up and release, the gather arguments, the prologue of a step (prep,
// prioritised draw, gather, gradient zeroing, forward launches) and its optimiser arguments, and the bodies of the replay,
// normalisation, step, training-state and metrics-log entry points.  A handle type derives from QLearner and brings its
// network, tail kernel and actor; `A` is its action width in floats per transition (BDQ: one bin per branch, DQN: 1).
// The observe path (b2g_*_observe_act / _add) is shared too: VecNormalize's obs_rms on the device (ObsRms, obsnorm.cuh), the
// staged current observations, and the commit of a call's transitions into the replay.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <functional>
#include <string>
#include <vector>

#include "../../include/b200grasp.h"
#include "common.cuh"
#include "host.cuh"
#include "metrics_log.cuh"
#include "obsnorm.cuh"
#include "per.cuh"
#include "state.cuh"

namespace b2g {

struct QLearner {
  // configuration
  int device = 0, rank = 0, nranks = 1;
  unsigned long long seed = 0;        // the caller's seed; the Philox key of the replay draw mixes the rank into it (philox_key)
  float gamma = 0.f;
  int B = 0, E = 0, XS = 0, A = 1;    // batch, observation width, gathered row stride, action width
  int64_t buffer_capacity = 0;
  bool prioritized = false;
  float per_alpha = 0.f, per_eps = 0.f;
  // parameters: the zip's variables, the online tensors then their target copies at off + n_train
  ParamTable params;
  int64_t n_train = 0;
  float *P = nullptr, *Mo = nullptr, *Vo = nullptr, *G = nullptr, *metrics = nullptr;
  float eps_value = 1.0f;             // the zip's exploration epsilon variable
  cudaStream_t stream = nullptr;
  std::vector<void*> allocs;
  TransitionReplay replay;
  double *d_mean = nullptr, *d_istd = nullptr, *d_normc = nullptr;
  float *X = nullptr, *Xn = nullptr, *Xscratch = nullptr;
  float* td = nullptr;                // [B][A]
  float *rew_n = nullptr, *done_n = nullptr, *weights = nullptr, *eps_dummy = nullptr;
  float *s_obs = nullptr, *s_next = nullptr, *s_act = nullptr, *s_rew = nullptr, *s_done = nullptr;   // explicit batch
  int* indices = nullptr;
  int* act_idx_out = nullptr;         // [B][A]
  long long* counters = nullptr;
  double* step_consts = nullptr;
  float* d_lr = nullptr;
  float cur_lr = -1.f;
  std::vector<GemmGroup> fwd, bwd, act;
  long long n_updates = 0;
  float* h_met = nullptr;             // pinned, MET_COUNT floats
  cudaGraphExec_t graph_exec = nullptr;
  bool use_graph = true;
  bool broken = false;                // a training-state load failed after it began writing: only destroy / load are accepted
  MetricsLog mlog;                    // per-step metrics ring (b2g_*_metrics_log); off: the step has no append node
  // the observe path.  The obsnorm.cuh templates are instantiated on QLearner and read cfg, allocs, stream, stage_rows and ob_n
  // (a handle's own cfg hides this view).
  struct { int device = 0, nranks = 1; } cfg;
  const char* abi = "";               // "bdq" / "dqn": the b2g_<abi>_* entry points named in error text
  ObsRms rms;                         // device VecNormalize statistics (b2g_*_obs_rms_set), upload counts, observation encoder
  // b2g_*_observe_act / _add staging (allocated on first use): the current observation of env i as a row of ob_rows[ob_k] (the
  // other buffer takes the next call's next_obs), the reset frames of finished envs, and the call's actions / rewards / done flags.
  int stage_rows = 0;                 // envs per observe call
  float* ob_rows[2]{};                // [stage_rows + B][E] (the actor's gather reads B rows from any chunk start)
  float* ob_reset = nullptr;          // [stage_rows][E]
  float *ob_act = nullptr, *ob_rew = nullptr, *ob_done = nullptr;
  int* ob_idx = nullptr;              // [stage_rows][A] actor output
  int ob_k = 0, ob_n = 0;
  std::vector<int64_t> ob_fid;        // replay with frames: frame id holding env i's staged observation (-1: not stored yet)
  float* p(const std::string& nm) { return P + params.off(nm); }
  float* g(const std::string& nm) { return G + params.off(nm); }
  unsigned long long philox_key() const { return seed + 0x9E3779B97F4A7C15ull * (unsigned long long)rank; }
};

// After the configuration fields, the parameter table and n_train are set: B2G_NO_GRAPH, the stream, every QLearner buffer
// (G with g_extra floats more), the replay (frame_capacity of `replay`, stage_rows rows per commit and per observe call), the
// identity normalisation table and obs_rms's view of it, synchronously.
int ql_init(QLearner* h, int64_t g_extra, const b2g_replay_cfg* replay, int stage_rows);
// Frees what the handle holds (not h itself).
void ql_release(QLearner* h);

GatherArgs ql_gather(QLearner* h, bool from_replay, bool with_next);
// The start of a step on h->stream: prep (a uniform draw when sampled), the prioritised draw (then *weights = h->weights), the
// gather, zeroing g_floats floats of G and the forward groups.  *pr receives the PER arguments of the later priority update.
int ql_issue_prologue(QLearner* h, bool sampled, bool apply, size_t g_floats, const float** weights, PerArgs* pr);
// update_priorities(|td| + eps) after a sampled step with PER
void ql_issue_priorities(QLearner* h, bool sampled, const PerArgs& pr);
OptimArgs ql_optim_args(QLearner* h, bool apply);
// MET_COUNT metrics -> h->h_met, synchronising the stream
int ql_fetch(QLearner* h);

// ---- entry-point bodies; check(), when given, runs after the handle and argument checks and before anything is stored
int ql_replay_add(QLearner* h, const float* obs, const float* act, const float* rew, const float* next_obs, const float* done, int64_t n,
                  const std::function<int()>& check);
int64_t ql_replay_size(const QLearner* h);
int ql_replay_info(const QLearner* h, int64_t* capacity, int64_t* size, int64_t* frame_capacity, int64_t* live_frames, int64_t* bytes,
                   int64_t* evicted_early);
int ql_replay_get(QLearner* h, int64_t slot, float* obs, float* act, float* rew, float* next_obs, float* done, int32_t* frame_ids);
// rms: the handle's device obs_rms
int ql_set_norm_stats(QLearner* h, ObsRms* rms, const double* obs_mean, const double* obs_var, double ret_var, double clip_obs,
                      double clip_rew, double eps, int norm_obs, int norm_reward);
int ql_set_per_beta(QLearner* h, float beta);
int ql_get_last_per(QLearner* h, int32_t* slots, float* weights, float* priorities);
// n_steps sampled steps through the step graph (captured on the first call) or issue() under B2G_NO_GRAPH=1
int ql_step(QLearner* h, int n_steps, float lr, const std::function<int()>& issue);
// the explicit batch staged, then issue(apply, weights) and td_out [B][A]
int ql_step_explicit(QLearner* h, const float* obs, const float* act, const float* rew, const float* next_obs, const float* done,
                     const float* weights, float lr, int apply_update, float* td_out, const std::function<int()>& check,
                     const std::function<int(bool, const float*)>& issue);
// ---- the observe path (b2g_*_observe_act / _add; the handle is checked by the caller)
// observe_act without its actor: the refusals, the staging of n raw frames (obs != null: uploaded or encoded, merged into
// obs_rms when update_stats), then act(cur) on the staged rows [n][E] when acting; synchronises the stream once.
int ql_observe_act(QLearner* h, const float* obs, int n, int update_stats, bool acting, const std::function<int(const float*)>& act);
// observe_add: transition i = (staged obs_i, act_i [A], rew_i, next_obs_i, done_i) into the replay, as replay_add stores it,
// then next_obs (reset_obs where done) merged and staged.  check(), when given, runs after the refusals and before any CUDA work.
int ql_observe_add(QLearner* h, const float* act, const float* rew, const float* next_obs, const float* done, const float* reset_obs,
                   int n, int update_stats, const std::function<int()>& check);
// set_obs_encoder's body
int ql_set_obs_encoder(QLearner* h, const b2g_encoder* enc, int tail);
// ---- training state (container format in state.cuh).  refusal: the text of a B2G_ESTATE refusal of every state file, or null.
// rms: the handle's obs_rms section, or null.  restore() puts back what the handle keeps outside the shared fields.
int ql_state_save(QLearner* h, const char* path, uint32_t kind, const std::vector<FpField>& fp, ObsRms* rms, const char* refusal);
int ql_state_load(QLearner* h, const char* path, uint32_t kind, const std::vector<FpField>& fp, ObsRms* rms, const char* refusal,
                  const char* learner, const std::function<void()>& restore);
int ql_metrics_log(QLearner* h, int capacity, int cols);
// fix: the handle's host-side finishing of a row (as its fetch)
int ql_metrics_drain(QLearner* h, float* rows, int max_rows, int64_t* first_step, int* n_rows, int64_t* lost,
                     const std::function<void(float*)>& fix);

}  // namespace b2g
