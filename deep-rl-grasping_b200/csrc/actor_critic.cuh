// The actor-critic MLP that the PPO2 (ppo.cu) and TRPO (trpo.cu) handles share (common.policies.MlpPolicy: tanh towers pi and
// vf of widths [h0, h1] on the flattened observation, a state-independent pi/logstd and the untrained head q), its rollout of
// T steps of E envs, and what both handles do with them (actor_critic.cu): the parameter arena and the zip's table, the
// forward builder, the bias-tanh, actor and GAE kernels, the rollout and predict entry points and the training-state file.
// TRPO's rollout is this rollout with E = 1 and T = timesteps_per_batch.
//
// Both towers' first layers are one [D, 2 h0] matrix (pi columns, then vf columns), so layer 0 is one contraction over the
// shared input.  Arena order: W0, b0, W1 pi, b1 pi, W1 vf, b1 vf, vf/w, vf/b, pi/w, pi/b, pi/logstd (the trained block), then
// q/w, q/b.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <map>
#include <string>
#include <vector>

#include "common.cuh"
#include "host.cuh"
#include "obsnorm.cuh"
#include "state.cuh"

namespace b2g {

constexpr int kAcMaxA = 16;           // action components: the kernels keep a row's mean in registers
constexpr int kAcMaxWidth = 256;      // hidden widths (multiples of 4: 16-byte rows for the engine)
constexpr int kAcActThreads = 1024;
constexpr int kAcHostFloats = 64;     // the pinned h_buf

// Sum over the block in a fixed order: the same value on every call.  red holds one T per warp.
template <class T>
__device__ __forceinline__ T block_sum_t(T v, T* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  T t = 0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
  __syncthreads();
  return t;
}

struct AcHeadArgs {
  const float* Y1; int h1;             // [rows, 2 h1]: pi latent | vf latent
  const float* Wpi; const float* bpi;  // [h1, A], [A]
  const float* Wvf; const float* bvf;  // [h1, 1], [1]
  const float* logstd;                 // [A]
  int A;
};

// mean and value of row r
__device__ __forceinline__ void ac_heads(const AcHeadArgs& a, int r, float* mu, float& v) {
  const float* ypi = a.Y1 + (size_t)r * 2 * a.h1;
  const float* yvf = ypi + a.h1;
#pragma unroll
  for (int k = 0; k < kAcMaxA; ++k) mu[k] = k < a.A ? a.bpi[k] : 0.f;
  v = a.bvf[0];
  for (int j = 0; j < a.h1; ++j) {
    const float yp = ypi[j];
    const float* w = a.Wpi + (size_t)j * a.A;
#pragma unroll
    for (int k = 0; k < kAcMaxA; ++k)
      if (k < a.A) mu[k] = fmaf(yp, w[k], mu[k]);
    v = fmaf(yvf[j], a.Wvf[j], v);
  }
}

// Actor over `rows` rows.  mode 0: rollout step t (noise of stream 1, stores action / value / neglogp in row t and the actions
// in out); mode 1: values -> lastv; mode 2: predict (deterministic or stream-1 noise) -> out, values -> vout.
struct AcActArgs {
  AcHeadArgs h;
  int rows, mode, deterministic, t;
  unsigned long long key;
  long long* step;                     // stream-1 step counter (advanced by one per drawing call)
  float* r_act; float* r_val; float* r_nlp;   // rollout rows
  float* lastv;
  float* out; float* vout; float* nlpout;
};

// one forward pass (layers 0 and 1 of both towers) over M rows of an observation arena
struct AcFwd { GemmGroup l0, l1; int M = 0; };

using AcTab = std::map<std::string, const int*>;

// The network, rollout and bookkeeping of one handle.  A handle type derives from it; ac_init, ac_layout and ac_alloc fill it.
struct ActorCritic {
  int device = 0;
  int D = 0, XS = 0, A = 0, H0 = 0, H1 = 0;
  int E = 0, T = 0, P_ROWS = 0;       // rollout of T steps of E envs; predict chunks of P_ROWS rows
  int64_t oW0 = 0, ob0 = 0, oW1[2]{}, ob1[2]{}, oWvf = 0, obvf = 0, oWpi = 0, obpi = 0, ols = 0;
  int64_t n_train = 0, n_total = 0;   // the trained block; the whole network (q included)
  int64_t n_param = 0;                // floats of the parameter arena (n_total, or more when the handle keeps copies)
  ParamTable params;                  // the zip's variables
  float* P = nullptr;                 // parameter arena
  float *G = nullptr, *Mo = nullptr, *Vo = nullptr;   // gradient arena and Adam moments, n_train floats each
  cudaStream_t stream = nullptr;
  std::vector<void*> allocs;
  // rollout: rows of E observations (stride XS), actions, values, neglogp, rewards, episode-start flags, GAE outputs; row T
  // holds the observations after the last step (and the values / actions / neglogp drawn there)
  float *r_obs = nullptr, *r_act = nullptr, *r_val = nullptr, *r_nlp = nullptr, *r_rew = nullptr, *r_done = nullptr;
  float *r_adv = nullptr, *r_ret = nullptr, *lastv = nullptr;
  int t = 0;                          // rollout rows filled
  float* p_obs = nullptr;             // predict staging, P_ROWS rows
  int* act_rowoff = nullptr;          // the actor's E row offsets
  // activations of the forward builder (enough rows for every forward of the handle)
  float *Z0 = nullptr, *Y0 = nullptr, *Y1 = nullptr;
  float *a_out = nullptr, *a_v = nullptr, *a_nlp = nullptr;   // actor outputs
  long long* counters = nullptr;      // [4]: [0] Adam step, [1] the stream-1 step, then the handle's own
  unsigned long long act_key = 0;
  float* h_buf = nullptr;             // pinned, kAcHostFloats
  AcFwd f_act, f_boot, f_pred;        // the rollout step, the bootstrap row T, predict
  cudaGraphExec_t graph_exec = nullptr;
  bool use_graph = true;
  bool broken = false;
  long long n_updates = 0;
  bool acted = false;                 // row t's action is drawn: an observation staged now belongs to row t + 1
  // VecNormalize's obs_rms on the device (ObsRms, obsnorm.cuh) and the observe path that normalises each frame once into the
  // rollout.  The obsnorm.cuh templates are instantiated on ActorCritic and read cfg, allocs, stream, stage_rows and ob_n (a
  // handle's own cfg hides this one).
  ObsRms rms;
  struct { int device = 0, nranks = 1; } cfg;
  double clip_obs = 10.0;             // VecNormalize.clip_obs of the last set_norm_stats
  bool norm_obs = true;               // VecNormalize.norm_obs: false copies the rows as they are
  int stage_rows = 0;                 // E: the rows of an observe call (and of the encoder stage)
  int ob_n = 0, ob_row = -1;          // ob_n observations staged (0 or E), normalised into rollout row ob_row
  float* ob_stage = nullptr;          // [max(E, P_ROWS)][D] frames as uploaded or encoded, before the normalisation
  double* rms_tab = nullptr;          // [2][D]: the d_mean / d_istd table ObsRms::merge rewrites (nothing here reads it)
};

// The configuration checks both handles make first: obs_dim, n_actions and the hidden widths.
int ac_check_net(int obs_dim, int n_actions, int hidden0, int hidden1);
inline int64_t ac_row_stride(int obs_dim) { return (obs_dim + 3) / 4 * 4; }
// Shapes, the actor key (oracle/philox_ref.py act_seed), B2G_NO_GRAPH and the stream.
int ac_init(ActorCritic* h, int device, int D, int A, int H0, int H1, int E, int T, int p_rows, uint64_t seed);
// The arena offsets, n_train / n_total / n_param = n_total * copies, and the zip's 15 entries under scope in their order; entry i
// is in the gradient arena when bit i of grad_mask is set.
void ac_layout(ActorCritic* h, const std::string& scope, uint32_t grad_mask, int copies);
// The storage of every ActorCritic field (activations for `rows` rows), the offset tables iD, iH0, iH1, i2H0, rM_2H0, rM_2H1,
// iH0_H1, iD_2H0, boot and pred into tab, and f_act / f_boot / f_pred.
int ac_alloc(ActorCritic* h, int rows, AcTab& tab);
// Frees what the handle holds (not h itself).
void ac_release(ActorCritic* h);

// split-R so a launch covers about two waves of the 132 SMs, >= 64 rows per slice
int ac_splits_for(int tiles, int R);
// Layers 0 and 1 over M rows of `obs` at row offsets rowoff, into Z0 / Y0 / Y1, with the tables of ac_alloc.
int ac_make_fwd(ActorCritic* h, AcFwd& f, const float* obs, const int* rowoff, int M, AcTab& tab);
void ac_fwd_issue(ActorCritic* h, const AcFwd& f, cudaStream_t s);
// Y[i] = tanh(Z[i] + b[i % N]) over n rows of N columns
void ac_bias_tanh(const float* Z, const float* b, float* Y, int n, int N, cudaStream_t s);
AcHeadArgs ac_head_args(const ActorCritic* h);
AcActArgs ac_act_args(ActorCritic* h, int rows, int mode);
void ac_act(const AcActArgs& a, cudaStream_t s);
// GAE (ppo2.py Runner._run, trpo_mpi/utils.py add_vtarg_and_adv): a thread per env, reverse over the T rows.  done[t] is the
// episode-start flag of step t, done[T] the flags after the last step.
void ac_gae(const float* rew, const float* val, const float* done, const float* lastv, int T, int E, float gamma, float lam, float* adv,
            float* ret, cudaStream_t s);

// ---- entry-point bodies (the caller has checked the handle and its arguments)
int ac_upload_rows(ActorCritic* h, float* dst, const float* src, int rows);   // [rows, D] -> rows of stride XS
// E observations into row t; the forward pass and the actor's draw of step t -> act_out [E, A]
int ac_rollout_act(ActorCritic* h, const float* obs, float* act_out);
// row t's E rewards and the next episode-start flags; t += 1
int ac_rollout_reward(ActorCritic* h, const float* rew, const float* done);
int ac_rollout_reset(ActorCritic* h);
int ac_rollout_get(ActorCritic* h, float* adv, float* ret, float* val, float* nlp, float* act);   // nulls are skipped
// issue() through the update graph (captured on the first call) or directly under B2G_NO_GRAPH=1
int ac_run_update(ActorCritic* h, const std::function<int()>& issue);
// in chunks of P_ROWS rows; value_out and nlp_out may be null.  raw: the rows are normalised with the current obs_rms first
// (nothing is merged)
int ac_predict(ActorCritic* h, const float* obs, int n, int deterministic, float* act_out, float* value_out, float* nlp_out,
               bool raw = false);
int ac_get_step(ActorCritic* h, int64_t* adam_step, int64_t* noise_step, int32_t* rollout_rows);

// ---- VecNormalize's obs_rms on the device and the observe path (b2g_ppo_* / b2g_trpo_* forward to these)
// n rows [n][D] at x -> rows of stride XS at dst: float(clip((double(x) - mean) / sqrt(var + eps), -clip_obs, clip_obs)) in
// float64, numpy's order, rounded once; a copy without obs_rms or with norm_obs off; the pad columns [D, XS) are zero
void ac_obs_normalize(const ActorCritic* h, const float* x, int n, float* dst, cudaStream_t s);
int ac_obs_rms_set(ActorCritic* h, const double* mean, const double* var, double count);
int ac_obs_rms_get(ActorCritic* h, double* mean, double* var, double* count);
int ac_upload_bytes(const ActorCritic* h, int64_t* observe_bytes, int64_t* other_bytes);
int ac_set_norm_stats(ActorCritic* h, double clip_obs, double eps, int norm_obs);
int ac_set_obs_encoder(ActorCritic* h, const b2g_encoder* enc, int tail);
// obs: n = E raw frames uploaded once, merged when update_stats, normalised into the current row (t, or t + 1 once row t's
// action is drawn); act_out: the rollout step on row t.  carried: row 0 holds an action drawn before the last update (TRPO's
// boundary), returned without a draw.  One stream synchronise.
int ac_observe_act(ActorCritic* h, const float* obs, int n, int update_stats, float* act_out, bool carried);
// update's last_obs: uploaded into row T, or NULL: the row observe_act staged there (the check: B2G_EINVAL without one)
int ac_check_last_obs(const ActorCritic* h, const float* last_obs);
int ac_update_last_obs(ActorCritic* h, const float* last_obs);
// after an update's launch: with a staged row T it is the first observation of the next rollout, in row 0 (copy_row0: the
// update did not copy it there itself)
int ac_update_finish(ActorCritic* h, const float* last_obs, bool copy_row0);

// ---- debug read-back (b2g_debug_ppo_tensor / b2g_debug_trpo_tensor): one named device buffer, its element count and size
struct AcDebugBuf { const void* p = nullptr; int64_t numel = 0; int elem_bytes = 4; };
// The ActorCritic fields (activations of `rows` rows): P G Mo Vo Z0 Y0 Y1 r_obs r_act r_val r_nlp r_rew r_done r_adv r_ret
// lastv a_out a_v a_nlp act_rowoff counters.  false for any other name.
bool ac_debug_base(const ActorCritic* h, int rows, const std::string& name, AcDebugBuf& b);
// The bodies of the _info and read entry points; find fills b or fails with the unknown name.  The read syncs the handle's stream.
int ac_debug_info(const AcDebugBuf& b, int64_t* numel, int32_t* elem_bytes);
int ac_debug_read(ActorCritic* h, const AcDebugBuf& b, const char* name, void* dst, size_t bytes);

// ---- training state (container format in state.cuh): HOST {n_updates, 0}, CNTR the 4 counters, then the parameter arena and
// the Adam moments, then ORMS (obs_rms) behind the obs_rms fingerprint field when the handle owns device statistics.  An
// update boundary: the rollout in flight is not saved; a load leaves an empty rollout with cleared episode-start flags and
// nothing staged (the env starts a fresh episode).
int ac_state_save(ActorCritic* h, const char* path, uint32_t kind, const std::vector<FpField>& fp);
int ac_state_load(ActorCritic* h, const char* path, uint32_t kind, const std::vector<FpField>& fp, const char* learner);

}  // namespace b2g
