// The actor-critic MLP that the PPO2 (ppo.cu) and TRPO (trpo.cu) handles share (common.policies.MlpPolicy: tanh towers pi and
// vf of widths [h0, h1] on the flattened observation, a state-independent pi/logstd and the untrained head q), and its
// single-env-or-more rollout storage: the forward builder, the bias-tanh, actor and GAE kernels (actor_critic.cu).
//
// Both towers' first layers are one [D, 2 h0] matrix (pi columns, then vf columns), so layer 0 is one contraction over the
// shared input.  Arena order: W0, b0, W1 pi, b1 pi, W1 vf, b1 vf, vf/w, vf/b, pi/w, pi/b, pi/logstd (the trained block), then
// q/w, q/b.
#pragma once
#include <cuda_runtime.h>

#include <map>
#include <string>
#include <vector>

#include "common.cuh"

namespace b2g {

constexpr int kAcMaxA = 16;           // action components: the kernels keep a row's mean in registers
constexpr int kAcMaxWidth = 256;      // hidden widths (multiples of 4: 16-byte rows for the engine)
constexpr int kAcActThreads = 1024;

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

// The network and rollout of one handle.  A handle type derives from it and fills every field at create time.
struct ActorCritic {
  int D = 0, XS = 0, A = 0, H0 = 0, H1 = 0;
  int64_t oW0 = 0, ob0 = 0, oW1[2]{}, ob1[2]{}, oWvf = 0, obvf = 0, oWpi = 0, obpi = 0, ols = 0;
  float* P = nullptr;                 // parameter arena
  cudaStream_t stream = nullptr;
  std::vector<void*> allocs;
  // rollout: rows of n_envs observations (stride XS), actions, values, neglogp, rewards, episode-start flags, GAE outputs
  float *r_obs = nullptr, *r_act = nullptr, *r_val = nullptr, *r_nlp = nullptr, *r_rew = nullptr, *r_done = nullptr;
  float *r_adv = nullptr, *r_ret = nullptr, *lastv = nullptr;
  int t = 0;                          // rollout rows filled
  // activations of the forward builder (enough rows for every forward of the handle)
  float *Z0 = nullptr, *Y0 = nullptr, *Y1 = nullptr;
  float *a_out = nullptr, *a_v = nullptr, *a_nlp = nullptr;   // actor outputs
  long long* counters = nullptr;      // [1]: the stream-1 step
  unsigned long long act_key = 0;
};

// one forward pass (layers 0 and 1 of both towers) over M rows of an observation arena
struct AcFwd { GemmGroup l0, l1; int M = 0; };

// split-R so a launch covers about two waves of the 132 SMs, >= 64 rows per slice
int ac_splits_for(int tiles, int R);
// Layers 0 and 1 over M rows of `obs` at row offsets rowoff, into Z0 / Y0 / Y1.  tab holds the offset tables iD, iH0, iH1,
// i2H0, rM_2H0, rM_2H1, iH0_H1 and iD_2H0.
int ac_make_fwd(ActorCritic* h, AcFwd& f, const float* obs, const int* rowoff, int M, std::map<std::string, const int*>& tab);
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

}  // namespace b2g
