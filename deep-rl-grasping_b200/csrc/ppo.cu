// libb200grasp: PPO2 learner -- the `sb.PPO2` branch of sb_helper.py:137-154 (stable-baselines 2.10.1 ppo2, restated in
// oracle/ppo_ref.py).
//
// Network (common/policies.py FeedForwardPolicy, net_arch=[dict(pi=[h0, h1], vf=[h0, h1])], tanh): two towers on the
// flattened observation, pi: obs -> h0 -> h1 -> mean [A], vf: obs -> h0 -> h1 -> value, a state-independent pi/logstd [1, A],
// and the head q (vf latent -> A) that nothing trains.  Both towers' first layers are one [D, 2 h0] matrix (pi columns, then
// vf columns), so layer 0 is one contraction over the shared input; get / set repack it to the zip's pi_fc0/w and vf_fc0/w.
//
// Rollout: b2g_ppo_rollout_act uploads the n_envs observations straight into rollout row t, runs the forward pass and draws
// mean + std * eps (Philox stream 1 under the caller's key at the device step counter); b2g_ppo_rollout_reward stores row t's
// rewards and the next episode-start flags.  Observations cross PCIe once.
//
// Update (b2g_ppo_update, one CUDA graph): bootstrap value of last_obs, GAE (a thread per env, reverse scan), then for each of
// noptepochs x nminibatches minibatches, in the caller's permutation:
//   layer 0   gather-GEMM through the permutation rows, split-R into Z0, then tanh(Z0 + b0)
//   layer 1   both towers, one grouped launch with the tanh epilogue
//   tail      one CTA: heads, minibatch advantage normalisation, clipped losses and metrics, head backward, head / logstd
//             gradients and dZ1 = (dY1)(1 - Y1^2)
//   layer 1   weight / bias gradients of both towers and dZ0 = dZ1 W1^T (1 - Y0^2), one grouped launch
//   layer 0   weight / bias gradient X^T dZ0 (D up to 20480 rows)
//   norm      global L2 norm of the gradient arena (fixed-order partials)
//   Adam      TF1 Adam, eps 1e-5, on g * min(1, max_grad_norm / norm)   (tf.clip_by_global_norm)
// q/w and q/b sit behind the trained arena: no gradient, no Adam moments.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "../../include/b200grasp.h"
#include "actor_critic.cuh"
#include "common.cuh"
#include "host.cuh"
#include "state.cuh"

using namespace b2g;

namespace {

constexpr int kMaxA = kAcMaxA;       // action components: the tail keeps a row's mean in registers
constexpr int kMaxMinibatch = 16384; // one tail CTA walks the minibatch
constexpr int kTailThreads = 1024;
constexpr int kNormBlocks = 128, kNormThreads = 256;
constexpr float kAdamEps = 1e-5f;    // ppo2.py: tf.train.AdamOptimizer(learning_rate, epsilon=1e-5)

// metric slots: the last minibatch [0, 8) and the sums over an update's minibatches [8, 16)
enum : int { PM_PG = 0, PM_VF, PM_ENT, PM_KL, PM_CLIP, PM_GN, PM_N = 8 };
// device hyper-parameters of the current call: lr, cliprange, cliprange_vf (< 0: no value clipping)
enum : int { HP_LR = 0, HP_CLIP, HP_CLIPVF, HP_N = 4 };

// ---------------------------------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------------------------------

// permutation -> storage rows: flattened (env-major) batch index f = e * n_steps + t lives in rollout row t * n_envs + e
__global__ void ppo_rows_kernel(const int* __restrict__ perm, int n, int n_steps, int n_envs, int XS, int* __restrict__ rowidx,
                                int* __restrict__ rowoff) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int f = perm[i], e = f / n_steps, t = f - e * n_steps;
  const int r = t * n_envs + e;
  rowidx[i] = r;
  rowoff[i] = r * XS;
}

struct TailArgs2 {
  AcHeadArgs h;
  int M;
  const int* rowidx;                           // minibatch row -> rollout / staging row
  const float* act; const float* oval; const float* onlp; const float* ret;
  const float* hp;                             // HP_* device scalars
  float ent_coef, vf_coef;
  float* sz; float* sv; float* snlp; float* sadv; float* sdm; float* sdls; float* sdv;   // scratch [M] / [M, A]
  float* dZ1;                                  // [M, 2 h1]
  float* gWpi; float* gbpi; float* gWvf; float* gbvf; float* glogstd;
  float* met;                                  // PM_* slots [0, 8) last, [8, 16) sums
};

// ppo2.py _train_step on one minibatch, after layer 1: heads, the clipped losses and their gradients down to dZ1
__global__ void __launch_bounds__(kTailThreads) ppo_tail_kernel(TailArgs2 a) {
  __shared__ float red[kTailThreads / 32];
  const int M = a.M, A = a.h.A, h1 = a.h.h1, tid = threadIdx.x, NT = blockDim.x;
  const float clip = a.hp[HP_CLIP], clipvf = a.hp[HP_CLIPVF];
  const float invM = 1.0f / (float)M;
  // ---- heads, neglogp, raw advantages
  float s = 0.f;
  for (int r = tid; r < M; r += NT) {
    const int q = a.rowidx[r];
    float mu[kMaxA], v;
    ac_heads(a.h, r, mu, v);
    float nlp = 0.91893853320467274f * (float)A;
    for (int k = 0; k < A; ++k) {
      const float ls = a.h.logstd[k];
      const float z = (a.act[(size_t)q * A + k] - mu[k]) / expf(ls);
      a.sz[(size_t)r * A + k] = z;
      nlp += 0.5f * z * z + ls;
    }
    const float adv = a.ret[q] - a.oval[q];
    a.sv[r] = v; a.snlp[r] = nlp; a.sadv[r] = adv;
    s += adv;
  }
  const float mean = block_sum_t(s, red) * invM;
  float ss = 0.f;
  for (int r = tid; r < M; r += NT) { const float d = a.sadv[r] - mean; ss += d * d; }
  const float stdv = sqrtf(block_sum_t(ss, red) * invM);        // np.std: population
  // ---- losses and the gradient seeds
  float pg_s = 0.f, vf_s = 0.f, kl_s = 0.f, cf_s = 0.f;
  for (int r = tid; r < M; r += NT) {
    const int q = a.rowidx[r];
    const float advn = (a.sadv[r] - mean) / (stdv + 1e-8f);
    const float onlp = a.onlp[q], nlp = a.snlp[r];
    const float ratio = expf(onlp - nlp);
    const float lo = 1.f - clip, hi = 1.f + clip;
    const float rc = fminf(fmaxf(ratio, lo), hi);
    const float pg1 = -advn * ratio, pg2 = -advn * rc;
    pg_s += fmaxf(pg1, pg2);
    // tf.maximum sends the gradient to its first argument on ties; tf.clip_by_value passes it inside [lo, hi]
    const float dratio = (pg1 >= pg2 || (ratio >= lo && ratio <= hi)) ? -advn : 0.f;
    const float g_nlp = -dratio * ratio * invM;
    const float v = a.sv[r], R = a.ret[q], ov = a.oval[q];
    float l1 = (v - R) * (v - R), dv = (v - R);
    if (clipvf >= 0.f) {
      const float d = v - ov, vc = ov + fminf(fmaxf(d, -clipvf), clipvf);
      const float l2 = (vc - R) * (vc - R);
      if (l2 > l1) { l1 = l2; dv = (d >= -clipvf && d <= clipvf) ? (vc - R) : 0.f; }
    }
    vf_s += l1;
    a.sdv[r] = a.vf_coef * dv * invM;
    kl_s += (nlp - onlp) * (nlp - onlp);
    cf_s += fabsf(ratio - 1.f) > clip ? 1.f : 0.f;
    for (int k = 0; k < A; ++k) {
      const float z = a.sz[(size_t)r * A + k];
      a.sdm[(size_t)r * A + k] = -g_nlp * z / expf(a.h.logstd[k]);   // d nlp / d mu = -z / sigma
      a.sdls[(size_t)r * A + k] = g_nlp * (1.f - z * z);             // d nlp / d logstd = 1 - z^2
    }
  }
  const float pg = block_sum_t(pg_s, red) * invM, vfl = 0.5f * block_sum_t(vf_s, red) * invM;
  const float kl = 0.5f * block_sum_t(kl_s, red) * invM, cf = block_sum_t(cf_s, red) * invM;
  __syncthreads();                                                    // sdm / sdls / sdv of every row are written
  // ---- head backward: dZ1 = dY1 (1 - Y1^2) for both towers
  for (int i = tid; i < M * h1; i += NT) {
    const int r = i / h1, k = i - r * h1;
    const float* dm = a.sdm + (size_t)r * A;
    const float* w = a.h.Wpi + (size_t)k * A;
    float d = 0.f;
    for (int j = 0; j < A; ++j) d = fmaf(dm[j], w[j], d);
    const float yp = a.h.Y1[(size_t)r * 2 * h1 + k], yv = a.h.Y1[(size_t)r * 2 * h1 + h1 + k];
    a.dZ1[(size_t)r * 2 * h1 + k] = d * (1.f - yp * yp);
    a.dZ1[(size_t)r * 2 * h1 + h1 + k] = a.sdv[r] * a.h.Wvf[k] * (1.f - yv * yv);
  }
  // ---- head and logstd gradients: sums over the minibatch, one output per thread
  const int n_wpi = h1 * A, n_jobs = n_wpi + A + h1 + 1 + A;
  for (int jb = tid; jb < n_jobs; jb += NT) {
    float g = 0.f;
    if (jb < n_wpi) {
      const int k = jb / A, j = jb - k * A;
      for (int r = 0; r < M; ++r) g = fmaf(a.h.Y1[(size_t)r * 2 * h1 + k], a.sdm[(size_t)r * A + j], g);
      a.gWpi[jb] = g;
    } else if (jb < n_wpi + A) {
      const int j = jb - n_wpi;
      for (int r = 0; r < M; ++r) g += a.sdm[(size_t)r * A + j];
      a.gbpi[j] = g;
    } else if (jb < n_wpi + A + h1) {
      const int k = jb - n_wpi - A;
      for (int r = 0; r < M; ++r) g = fmaf(a.h.Y1[(size_t)r * 2 * h1 + h1 + k], a.sdv[r], g);
      a.gWvf[k] = g;
    } else if (jb == n_wpi + A + h1) {
      for (int r = 0; r < M; ++r) g += a.sdv[r];
      a.gbvf[0] = g;
    } else {
      const int j = jb - (n_wpi + A + h1 + 1);
      for (int r = 0; r < M; ++r) g += a.sdls[(size_t)r * A + j];
      a.glogstd[j] = g - a.ent_coef;                  // loss = ... - ent_coef * mean sum(logstd + .5 log(2 pi e))
    }
  }
  if (tid == 0) {
    float ent = 1.4189385332046727f * (float)A;     // 0.5 log(2 pi e) per component
    for (int k = 0; k < A; ++k) ent += a.h.logstd[k];
    const float m[5] = {pg, vfl, ent, kl, cf};
    for (int k = 0; k < 5; ++k) { a.met[k] = m[k]; a.met[PM_N + k] += m[k]; }
  }
}

// squared L2 norm of the gradient arena: fixed grid, one partial per CTA; the block also advances the Adam step
__global__ void __launch_bounds__(kNormThreads) ppo_norm_kernel(const float* __restrict__ G, int n4, float* __restrict__ part,
                                                                long long* counters) {
  __shared__ float red[kNormThreads / 32];
  float s = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
    const float4 g = reinterpret_cast<const float4*>(G)[i];
    s += g.x * g.x + g.y * g.y + g.z * g.z + g.w * g.w;
  }
  const float t = block_sum_t(s, red);
  if (threadIdx.x == 0) {
    part[blockIdx.x] = t;
    if (blockIdx.x == 0) counters[0] += 1;
  }
}

// TF1 Adam (epsilon 1e-5) on the globally clipped gradient: g * max_norm / max(norm, max_norm) (tf.clip_by_global_norm)
__global__ void __launch_bounds__(256) ppo_adam_kernel(float* __restrict__ P, float* __restrict__ Mo, float* __restrict__ Vo,
                                                       float* __restrict__ G, int n4, const float* __restrict__ part,
                                                       const long long* counters, const float* hp, float max_norm, int apply,
                                                       float* met) {
  __shared__ float s_scale;
  __shared__ float s_lrt;
  if (threadIdx.x < 32) {
    float v = 0.f;
    for (int i = threadIdx.x; i < kNormBlocks; i += 32) v += part[i];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) {
      const float norm = sqrtf(v);
      s_scale = max_norm / fmaxf(norm, max_norm);
      const double t = (double)counters[0];
      s_lrt = (float)((double)hp[HP_LR] * sqrt(1.0 - pow(0.999, t)) / (1.0 - pow(0.9, t)));
      if (blockIdx.x == 0) { met[PM_GN] = norm; met[PM_N + PM_GN] += norm; }
    }
  }
  __syncthreads();
  const float sc = s_scale, lr = s_lrt, b1 = 0.9f, b2 = 0.999f;
  for (int i4 = blockIdx.x * blockDim.x + threadIdx.x; i4 < n4; i4 += gridDim.x * blockDim.x) {
    float4 g = reinterpret_cast<float4*>(G)[i4];
    g.x *= sc; g.y *= sc; g.z *= sc; g.w *= sc;
    reinterpret_cast<float4*>(G)[i4] = g;                 // b2g_ppo_get_grad reads the clipped gradient
    if (!apply) continue;
    float4 m = reinterpret_cast<float4*>(Mo)[i4], v = reinterpret_cast<float4*>(Vo)[i4], p = reinterpret_cast<float4*>(P)[i4];
#define B2G_PPO_ADAM(c)                              \
  m.c = b1 * m.c + (1.f - b1) * g.c;                 \
  v.c = b2 * v.c + (1.f - b2) * (g.c * g.c);         \
  p.c = p.c - lr * m.c / (sqrtf(v.c) + kAdamEps);
    B2G_PPO_ADAM(x) B2G_PPO_ADAM(y) B2G_PPO_ADAM(z) B2G_PPO_ADAM(w)
#undef B2G_PPO_ADAM
    reinterpret_cast<float4*>(Mo)[i4] = m;
    reinterpret_cast<float4*>(Vo)[i4] = v;
    reinterpret_cast<float4*>(P)[i4] = p;
  }
}

}  // namespace

// the backward launches of a minibatch after its forward pass
struct PpoMb { AcFwd f; GemmGroup b1, b0; const int* rowidx = nullptr; };

// network, rollout, actor, update graph, counters [0] Adam step, [1] stream-1 step (actor_critic.cuh); h_buf holds metrics and
// hyper-parameters
struct b2g_ppo : ActorCritic {
  b2g_ppo_cfg cfg{};
  int NB = 0, M = 0, NMB = 0, RMAX = 0;
  // explicit minibatch staging
  float *s_obs = nullptr, *s_act = nullptr, *s_val = nullptr, *s_nlp = nullptr, *s_ret = nullptr;
  // backward activations and scratch (RMAX rows)
  float *dZ1 = nullptr, *dZ0 = nullptr;
  float *sz = nullptr, *sv = nullptr, *snlp = nullptr, *sadv = nullptr, *sdm = nullptr, *sdls = nullptr, *sdv = nullptr;
  int *perm = nullptr, *rowidx = nullptr, *rowoff = nullptr;
  float *part = nullptr, *met = nullptr, *hp = nullptr;
  PpoMb mb_explicit;
  std::vector<PpoMb> mbs;
};

namespace {

constexpr uint32_t kGradMask = (1u << 13) - 1;   // the trained block: every zip entry but q/w and q/b

// the zip names carry the model/ scope; the bare names are accepted too
std::string scoped(const char* name) { return strncmp(name, "model/", 6) == 0 ? name : "model/" + std::string(name); }

int make_mb(b2g_ppo* h, PpoMb& mb, const float* obs, const int* rowoff, const int* rowidx, AcTab& tab) {
  const int M = h->M, D = h->D, H0 = h->H0, H1 = h->H1;
  if (int rc = ac_make_fwd(h, mb.f, obs, rowoff, M, tab)) return rc;
  mb.rowidx = rowidx;
  mb.b1 = GemmGroup(); mb.b0 = GemmGroup();
  mb.b1.name = "ppo_l1_bwd"; mb.b0.name = "ppo_l0_wgrad";
  for (int tw = 0; tw < 2; ++tw) {
    const int tiles = ((H0 + 63) / 64) * ((H1 + 63) / 64);
    GemmDesc w = gemm_desc(h->Y0 + tw * H0, tab["iH0"], tab["rM_2H0"], h->dZ1 + tw * H1, tab["rM_2H1"], tab["iH1"], h->G + h->oW1[tw],
                           tab["iH0_H1"], tab["iH1"], H0, H1, M, GG_COLSUM | GG_EPI_ATOMIC, ac_splits_for(tiles, M));
    w.colsum = h->G + h->ob1[tw];
    mb.b1.host.push_back(w);
    GemmDesc dg = gemm_desc(h->dZ1 + tw * H1, tab["rM_2H1"], tab["iH1"], h->P + h->oW1[tw], tab["iH1"], tab["iH0_H1"], h->dZ0 + tw * H0,
                            tab["rM_2H0"], tab["iH0"], M, H0, H1, GG_A_RVEC | GG_B_RVEC | GG_EPI_TANH_GRAD);
    dg.mask = h->Y0 + tw * H0;
    mb.b1.host.push_back(dg);
  }
  const int tiles0 = ((D + 63) / 64) * ((2 * H0 + 63) / 64);
  GemmDesc w0 = gemm_desc(obs, tab["iD"], rowoff, h->dZ0, tab["rM_2H0"], tab["i2H0"], h->G + h->oW0, tab["iD_2H0"], tab["i2H0"], D, 2 * H0, M,
                          GG_COLSUM | GG_EPI_ATOMIC, ac_splits_for(tiles0, M));
  w0.colsum = h->G + h->ob0;
  mb.b0.host.push_back(w0);
  if (int rc = finalize_tiles(mb.b1, h->allocs, h->stream)) return rc;
  return finalize_tiles(mb.b0, h->allocs, h->stream);
}

// one minibatch: forward, tail, backward, global norm, Adam
void mb_issue(b2g_ppo* h, const PpoMb& mb, const float* act, const float* oval, const float* onlp, const float* ret, bool apply) {
  cudaStream_t s = h->stream;
  cudaMemsetAsync(h->G, 0, (size_t)h->n_train * sizeof(float), s);
  ac_fwd_issue(h, mb.f, s);
  TailArgs2 t{};
  t.h = ac_head_args(h); t.M = h->M; t.rowidx = mb.rowidx;
  t.act = act; t.oval = oval; t.onlp = onlp; t.ret = ret; t.hp = h->hp;
  t.ent_coef = h->cfg.ent_coef; t.vf_coef = h->cfg.vf_coef;
  t.sz = h->sz; t.sv = h->sv; t.snlp = h->snlp; t.sadv = h->sadv; t.sdm = h->sdm; t.sdls = h->sdls; t.sdv = h->sdv; t.dZ1 = h->dZ1;
  t.gWpi = h->G + h->oWpi; t.gbpi = h->G + h->obpi; t.gWvf = h->G + h->oWvf; t.gbvf = h->G + h->obvf; t.glogstd = h->G + h->ols;
  t.met = h->met;
  ppo_tail_kernel<<<1, kTailThreads, 0, s>>>(t);
  gg_simt_launch_tanh(mb.b1.dev, (int)mb.b1.host.size(), mb.b1.total_tiles, s);
  gg_simt_launch(mb.b0.dev, (int)mb.b0.host.size(), mb.b0.total_tiles, s);
  const int n4 = (int)(h->n_train / 4);
  ppo_norm_kernel<<<kNormBlocks, kNormThreads, 0, s>>>(h->G, n4, h->part, h->counters);
  ppo_adam_kernel<<<std::max(1, std::min(264, (n4 + 255) / 256)), 256, 0, s>>>(h->P, h->Mo, h->Vo, h->G, n4, h->part, h->counters, h->hp,
                                                                               h->cfg.max_grad_norm, apply ? 1 : 0, h->met);
}

// the whole update after the uploads: row map, bootstrap value, GAE, every minibatch
int update_issue(b2g_ppo* h) {
  cudaStream_t s = h->stream;
  const int n = h->cfg.noptepochs * h->NB;
  ppo_rows_kernel<<<(n + 255) / 256, 256, 0, s>>>(h->perm, n, h->T, h->E, h->XS, h->rowidx, h->rowoff);
  ac_fwd_issue(h, h->f_boot, s);
  ac_act(ac_act_args(h, h->E, 1), s);
  ac_gae(h->r_rew, h->r_val, h->r_done, h->lastv, h->T, h->E, h->cfg.gamma, h->cfg.lam, h->r_adv, h->r_ret, s);
  cudaMemsetAsync(h->met, 0, 2 * PM_N * sizeof(float), s);
  for (const PpoMb& mb : h->mbs) mb_issue(h, mb, h->r_act, h->r_val, h->r_nlp, h->r_ret, true);
  // the flags after the last step are the episode-start flags of the next rollout's first step
  cudaMemcpyAsync(h->r_done, h->r_done + (size_t)h->T * h->E, h->E * sizeof(float), cudaMemcpyDeviceToDevice, s);
  CK(cudaGetLastError());
  return 0;
}

int upload_hp(b2g_ppo* h, float lr, float clip, float clipvf) {
  if (!(lr >= 0.f) || !(clip >= 0.f)) return b2g_fail(B2G_EINVAL, "learning rate and cliprange must be >= 0");
  CK(cudaStreamSynchronize(h->stream));
  h->h_buf[0] = lr; h->h_buf[1] = clip; h->h_buf[2] = clipvf; h->h_buf[3] = 0.f;
  CK(cudaMemcpyAsync(h->hp, h->h_buf, HP_N * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  return 0;
}

int fetch(b2g_ppo* h, b2g_ppo_metrics* out, bool mean_of_update) {
  CK(cudaMemcpyAsync(h->h_buf, h->met, 2 * PM_N * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (out) {
    const float* m = mean_of_update ? h->h_buf + PM_N : h->h_buf;
    const float k = mean_of_update ? 1.0f / (float)h->mbs.size() : 1.0f;
    out->policy_loss = m[PM_PG] * k; out->value_loss = m[PM_VF] * k; out->entropy = m[PM_ENT] * k;
    out->approxkl = m[PM_KL] * k; out->clipfrac = m[PM_CLIP] * k; out->grad_norm = m[PM_GN] * k;
    out->n_updates = h->n_updates;
  }
  return 0;
}

}  // namespace

extern "C" {

int b2g_ppo_destroy(b2g_ppo* h) {
  if (!h) return 0;
  ac_release(h);
  delete h;
  return 0;
}

int b2g_ppo_create(const b2g_ppo_cfg* cfg, b2g_ppo** out) {
  if (!cfg || !out) return b2g_fail(B2G_EINVAL, "cfg/out is NULL");
  *out = nullptr;
  const b2g_ppo_cfg& c = *cfg;
  if (int rc = ac_check_net(c.obs_dim, c.n_actions, c.hidden0, c.hidden1)) return rc;
  if (c.n_envs < 1 || c.n_envs > 4096) return b2g_fail(B2G_EINVAL, "n_envs must be in [1, 4096]");
  if (c.n_steps < 1 || c.n_steps > 65536) return b2g_fail(B2G_EINVAL, "n_steps must be in [1, 65536]");
  if (c.nminibatches < 1 || c.noptepochs < 1) return b2g_fail(B2G_EINVAL, "nminibatches and noptepochs must be positive");
  const int64_t nb = (int64_t)c.n_steps * c.n_envs;
  if (nb % c.nminibatches) return b2g_fail(B2G_EINVAL, "n_batch = n_steps * n_envs must be divisible by nminibatches");
  if (nb / c.nminibatches > kMaxMinibatch) return b2g_fail(B2G_EINVAL, "minibatch n_batch / nminibatches must be <= 16384");
  if ((int64_t)c.noptepochs * c.nminibatches > 4096) return b2g_fail(B2G_EINVAL, "noptepochs * nminibatches must be <= 4096");
  const int64_t XS = ac_row_stride(c.obs_dim);
  if ((nb + c.n_envs) * XS >= (1LL << 31)) return b2g_fail(B2G_EINVAL, "rollout (n_steps + 1) * n_envs * obs_dim must be < 2^31 floats");
  if (int rc = check_device(c.device)) return rc;
  b2g_ppo* h = new b2g_ppo();
  h->cfg = c;
  auto bail = [&](int rc) { std::string keep = g_b2g_err; b2g_ppo_destroy(h); g_b2g_err = keep; return rc; };
  if (int rc = ac_init(h, c.device, c.obs_dim, c.n_actions, c.hidden0, c.hidden1, c.n_envs, c.n_steps, std::max(64, c.n_envs), c.seed))
    return bail(rc);
  h->rms.set_call = "b2g_ppo_obs_rms_set";
  h->NB = (int)nb; h->NMB = c.nminibatches; h->M = (int)(nb / c.nminibatches);
  h->RMAX = std::max(h->M, h->P_ROWS);
  ac_layout(h, "model/", kGradMask, 1);
  AcTab tab;
  int rc = ac_alloc(h, h->RMAX, tab);
  if (rc) return bail(rc);
  const int64_t A = h->A, H0 = h->H0, H1 = h->H1, R = h->RMAX;
#define DA(ptr, count) if ((rc = dev_alloc(h->allocs, h->stream, &(ptr), (size_t)(count)))) return bail(rc)
  DA(h->s_obs, (int64_t)h->M * XS); DA(h->s_act, (int64_t)h->M * A); DA(h->s_val, h->M); DA(h->s_nlp, h->M); DA(h->s_ret, h->M);
  DA(h->dZ1, R * 2 * H1); DA(h->dZ0, R * 2 * H0);
  DA(h->sz, R * A); DA(h->sv, R); DA(h->snlp, R); DA(h->sadv, R); DA(h->sdm, R * A); DA(h->sdls, R * A); DA(h->sdv, R);
  const int64_t nperm = (int64_t)c.noptepochs * h->NB;
  DA(h->perm, nperm); DA(h->rowidx, nperm); DA(h->rowoff, nperm);
  DA(h->part, kNormBlocks); DA(h->met, 2 * PM_N); DA(h->hp, HP_N);
#undef DA
  for (auto& [nm, v] : {std::make_pair("sM", iota_tab(h->M, h->XS)), std::make_pair("iM", iota_tab(h->M))}) {
    const int* p = nullptr;
    if ((rc = upload_table(h->allocs, h->stream, v, &p))) return bail(rc);
    tab[nm] = p;
  }
  if ((rc = make_mb(h, h->mb_explicit, h->s_obs, tab["sM"], tab["iM"], tab))) return bail(rc);
  h->mbs.resize((size_t)c.noptepochs * c.nminibatches);
  for (size_t k = 0; k < h->mbs.size(); ++k)
    if ((rc = make_mb(h, h->mbs[k], h->r_obs, h->rowoff + k * h->M, h->rowidx + k * h->M, tab))) return bail(rc);
  if (cudaStreamSynchronize(h->stream) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "create sync"));
  *out = h;
  return 0;
}

int b2g_ppo_param_count(const b2g_ppo* h) { return param_count(h); }
int b2g_ppo_param_info(const b2g_ppo* h, int idx, char* name, size_t name_cap, int64_t* rows, int64_t* cols, int32_t* ndim) {
  return param_info(h, idx, name, name_cap, rows, cols, ndim);
}
int b2g_ppo_get_param(b2g_ppo* h, const char* name, float* dst, size_t numel) {
  return param_copy(h, name ? scoped(name).c_str() : nullptr, ParamCopy::Get, dst, numel);
}
int b2g_ppo_set_param(b2g_ppo* h, const char* name, const float* src, size_t numel) {
  return param_copy(h, name ? scoped(name).c_str() : nullptr, ParamCopy::Set, const_cast<float*>(src), numel);
}
int b2g_ppo_get_grad(b2g_ppo* h, const char* name, float* dst, size_t numel) {
  return param_copy(h, name ? scoped(name).c_str() : nullptr, ParamCopy::GetGrad, dst, numel);
}

int b2g_ppo_rollout_act(b2g_ppo* h, const float* obs, float* act_out) {
  B2G_USABLE(h);
  if (!h || !obs || !act_out) return b2g_fail(B2G_EINVAL, "NULL argument");
  if (h->t >= h->T) return b2g_fail(B2G_ESTATE, "the rollout holds n_steps rows: call b2g_ppo_update first");
  return ac_rollout_act(h, obs, act_out);
}

int b2g_ppo_rollout_reward(b2g_ppo* h, const float* rew, const float* done) {
  B2G_USABLE(h);
  if (!h || !rew || !done) return b2g_fail(B2G_EINVAL, "NULL argument");
  if (h->t >= h->T) return b2g_fail(B2G_ESTATE, "the rollout holds n_steps rows: call b2g_ppo_update first");
  return ac_rollout_reward(h, rew, done);
}

int b2g_ppo_rollout_reset(b2g_ppo* h) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  return ac_rollout_reset(h);
}

int b2g_ppo_rollout_get(b2g_ppo* h, float* adv, float* ret, float* val, float* nlp, float* act) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  return ac_rollout_get(h, adv, ret, val, nlp, act);
}

int b2g_ppo_update(b2g_ppo* h, const float* last_obs, const int32_t* perm, float lr, float cliprange, float cliprange_vf,
                   b2g_ppo_metrics* out) {
  B2G_USABLE(h);
  if (!h || !perm) return b2g_fail(B2G_EINVAL, "NULL argument");
  if (h->t != h->T) return b2g_fail(B2G_ESTATE, "the rollout is not full: n_steps rollout steps come before an update");
  if (int rc = ac_check_last_obs(h, last_obs)) return rc;
  const int64_t n = (int64_t)h->cfg.noptepochs * h->NB;
  for (int64_t i = 0; i < n; ++i)
    if (perm[i] < 0 || perm[i] >= h->NB) return b2g_fail(B2G_EINVAL, "permutation entry " + std::to_string(i) + " is outside [0, n_batch)");
  CK(cudaSetDevice(h->cfg.device));
  if (int rc = upload_hp(h, lr, cliprange, cliprange_vf)) return rc;
  if (int rc = ac_update_last_obs(h, last_obs)) return rc;
  CK(cudaMemcpyAsync(h->perm, perm, n * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
  if (int rc = ac_run_update(h, [&] { return update_issue(h); })) return rc;
  h->n_updates += (int64_t)h->mbs.size();
  h->t = 0;
  if (int rc = ac_update_finish(h, last_obs, true)) return rc;
  return fetch(h, out, true);
}

int b2g_ppo_train_step_explicit(b2g_ppo* h, const float* obs, const float* returns, const float* actions, const float* values,
                                const float* neglogp, float lr, float cliprange, float cliprange_vf, int apply_update,
                                b2g_ppo_metrics* out) {
  B2G_USABLE(h);
  if (!h || !obs || !returns || !actions || !values || !neglogp) return b2g_fail(B2G_EINVAL, "NULL argument");
  CK(cudaSetDevice(h->cfg.device));
  if (int rc = upload_hp(h, lr, cliprange, cliprange_vf)) return rc;
  const size_t M = h->M;
  if (int rc = ac_upload_rows(h, h->s_obs, obs, h->M)) return rc;
  CK(cudaMemcpyAsync(h->s_ret, returns, M * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaMemcpyAsync(h->s_act, actions, M * h->A * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaMemcpyAsync(h->s_val, values, M * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaMemcpyAsync(h->s_nlp, neglogp, M * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaMemsetAsync(h->met, 0, 2 * PM_N * sizeof(float), h->stream));
  if (!apply_update) {    // the Adam step counter advances only with an applied step
    long long t0 = 0;
    CK(cudaMemcpyAsync(&t0, h->counters, sizeof t0, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    mb_issue(h, h->mb_explicit, h->s_act, h->s_val, h->s_nlp, h->s_ret, false);
    CK(cudaMemcpyAsync(h->counters, &t0, sizeof t0, cudaMemcpyHostToDevice, h->stream));
  } else {
    mb_issue(h, h->mb_explicit, h->s_act, h->s_val, h->s_nlp, h->s_ret, true);
    h->n_updates += 1;
  }
  CK(cudaGetLastError());
  return fetch(h, out, false);
}

int b2g_ppo_act(b2g_ppo* h, const float* obs, int n, int deterministic, float* act_out, float* value_out, float* neglogp_out) {
  B2G_USABLE(h);
  if (!h || !obs || !act_out || n < 0) return b2g_fail(B2G_EINVAL, "bad argument");
  return ac_predict(h, obs, n, deterministic, act_out, value_out, neglogp_out);
}

int b2g_ppo_get_step(b2g_ppo* h, int64_t* adam_step, int64_t* noise_step, int32_t* rollout_rows) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  return ac_get_step(h, adam_step, noise_step, rollout_rows);
}

// ---- VecNormalize's obs_rms on the device and the observe path (bodies in actor_critic.cu)
#define B2G_PPO_HANDLE(h) B2G_USABLE(h); if (!h) return b2g_fail(B2G_EINVAL, "NULL handle")
int b2g_ppo_obs_rms_set(b2g_ppo* h, const double* mean, const double* var, double count) { return ac_obs_rms_set(h, mean, var, count); }
int b2g_ppo_obs_rms_get(b2g_ppo* h, double* mean, double* var, double* count) { return ac_obs_rms_get(h, mean, var, count); }
int b2g_ppo_upload_bytes(const b2g_ppo* h, int64_t* observe_bytes, int64_t* other_bytes) { return ac_upload_bytes(h, observe_bytes, other_bytes); }
int b2g_ppo_set_norm_stats(b2g_ppo* h, double clip_obs, double eps, int norm_obs) { B2G_PPO_HANDLE(h); return ac_set_norm_stats(h, clip_obs, eps, norm_obs); }
int b2g_ppo_set_obs_encoder(b2g_ppo* h, const b2g_encoder* enc, int tail) { B2G_PPO_HANDLE(h); return ac_set_obs_encoder(h, enc, tail); }
int b2g_ppo_observe_act(b2g_ppo* h, const float* obs, int n, int update_stats, float* act_out) {
  B2G_PPO_HANDLE(h);
  return ac_observe_act(h, obs, n, update_stats, act_out, false);
}
int b2g_ppo_act_raw(b2g_ppo* h, const float* obs, int n, int deterministic, float* act_out, float* value_out, float* neglogp_out) {
  B2G_PPO_HANDLE(h);
  if (!obs || !act_out || n < 0) return b2g_fail(B2G_EINVAL, "bad argument");
  return ac_predict(h, obs, n, deterministic, act_out, value_out, neglogp_out, true);
}
#undef B2G_PPO_HANDLE

}  // extern "C"

// ================================================================================================
// Training state (b2g_ppo_state_save / _load; ac_state_save in actor_critic.cuh)
// ================================================================================================
namespace {

std::vector<FpField> ppo_fingerprint(const b2g_ppo* h) {
  const b2g_ppo_cfg& c = h->cfg;
  return {fp_int("obs_dim", c.obs_dim), fp_int("n_actions", c.n_actions), fp_int("hidden0", c.hidden0), fp_int("hidden1", c.hidden1),
          fp_int("n_envs", c.n_envs), fp_int("n_steps", c.n_steps), fp_int("nminibatches", c.nminibatches), fp_int("noptepochs", c.noptepochs),
          fp_int("seed", (int64_t)c.seed)};
}

}  // namespace

extern "C" {

int b2g_ppo_state_save(b2g_ppo* h, const char* path) {
  if (!h || !path) return b2g_fail(B2G_EINVAL, "NULL argument");
  B2G_USABLE(h);
  return ac_state_save(h, path, STATE_KIND_PPO, ppo_fingerprint(h));
}

int b2g_ppo_state_load(b2g_ppo* h, const char* path) {
  if (!h || !path) return b2g_fail(B2G_EINVAL, "NULL argument");
  return ac_state_load(h, path, STATE_KIND_PPO, ppo_fingerprint(h), "PPO2");
}

}  // extern "C"

// ================================================================================================
// Debug read-back of the handle's device buffers (b2g_debug_ppo_tensor; layouts in b200grasp.h)
// ================================================================================================
namespace {

int find_ppo_tensor(const b2g_ppo* h, const char* name, AcDebugBuf& b) {
  if (ac_debug_base(h, h->RMAX, name, b)) return 0;
  const int64_t R = h->RMAX, A = h->A, np = (int64_t)h->cfg.noptepochs * h->NB;
  const struct { const char* nm; const void* p; int64_t n; } t[] = {
      {"sz", h->sz, R * A},       {"sv", h->sv, R},           {"snlp", h->snlp, R},      {"sadv", h->sadv, R},
      {"sdm", h->sdm, R * A},     {"sdls", h->sdls, R * A},   {"sdv", h->sdv, R},        {"dZ1", h->dZ1, R * 2 * h->H1},
      {"dZ0", h->dZ0, R * 2 * h->H0}, {"part", h->part, kNormBlocks}, {"met", h->met, 2 * PM_N}, {"hp", h->hp, HP_N},
      {"rowidx", h->rowidx, np},  {"rowoff", h->rowoff, np},  {"perm", h->perm, np}};
  for (const auto& e : t)
    if (!strcmp(name, e.nm)) { b.p = e.p; b.numel = e.n; b.elem_bytes = 4; return 0; }
  return b2g_fail(B2G_EINVAL, std::string("unknown PPO2 debug tensor: ") + name);
}

}  // namespace

extern "C" {

int b2g_debug_ppo_tensor_info(const b2g_ppo* h, const char* name, int64_t* numel, int32_t* elem_bytes) {
  B2G_USABLE(h);
  if (!h || !name) return b2g_fail(B2G_EINVAL, "NULL argument");
  AcDebugBuf b;
  if (int rc = find_ppo_tensor(h, name, b)) return rc;
  return ac_debug_info(b, numel, elem_bytes);
}

int b2g_debug_ppo_tensor(b2g_ppo* h, const char* name, void* dst, size_t bytes) {
  B2G_USABLE(h);
  if (!h || !name || !dst) return b2g_fail(B2G_EINVAL, "NULL argument");
  AcDebugBuf b;
  if (int rc = find_ppo_tensor(h, name, b)) return rc;
  return ac_debug_read(h, b, name, dst, bytes);
}

}  // extern "C"
