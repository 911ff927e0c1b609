// The actor-critic MLP, its rollout and the handle code the PPO2 and TRPO handles share (actor_critic.cuh).
#include <cuda_runtime.h>
#include <math.h>
#include <stdlib.h>

#include <algorithm>
#include <cmath>
#include <string>

#include "actor_critic.cuh"

namespace b2g {

namespace {

__global__ void ppo_bias_tanh_kernel(const float* __restrict__ Z, const float* __restrict__ b, float* __restrict__ Y, int n, int N) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n * N) Y[i] = tanhf(Z[i] + b[i % N]);
}

__global__ void __launch_bounds__(kAcActThreads) ppo_act_kernel(AcActArgs a) {
  __shared__ unsigned long long s_step;
  const bool draw = a.mode == 0 || (a.mode == 2 && !a.deterministic);
  if (threadIdx.x == 0) s_step = (unsigned long long)*a.step;
  __syncthreads();
  const int A = a.h.A;
  const float half_log_2pi = 0.91893853320467274f;
  for (int r = threadIdx.x; r < a.rows; r += blockDim.x) {
    float mu[kAcMaxA], v;
    ac_heads(a.h, r, mu, v);
    if (a.mode == 1) { a.lastv[r] = v; continue; }
    float z[kAcMaxA];
#pragma unroll
    for (int k = 0; k < kAcMaxA; ++k) z[k] = 0.f;
    if (draw) {
      const uint2 key = make_uint2((unsigned)a.key, (unsigned)(a.key >> 32));
      // element r * A + k of the flattened [rows, A] noise: lane (i & 3) of block i >> 2 (oracle/philox_ref.py noise)
#pragma unroll
      for (int k = 0; k < kAcMaxA; ++k) {
        if (k >= A) break;
        const int i = r * A + k, blk = i >> 2;
        const uint4 q = philox4x32_10(make_uint4((unsigned)s_step, (unsigned)(s_step >> 32), (unsigned)blk, 1u), key);
        const int lane = i & 3;
        const unsigned x0 = lane < 2 ? q.x : q.z, x1 = lane < 2 ? q.y : q.w;
        const float u0 = ((float)(x0 >> 8) + 0.5f) * (1.0f / 16777216.0f), u1 = ((float)(x1 >> 8) + 0.5f) * (1.0f / 16777216.0f);
        const float rr = sqrtf(-2.f * logf(u0));
        float s, c;
        sincospif(2.f * u1, &s, &c);
        z[k] = rr * ((lane & 1) ? s : c);
      }
    }
    float nlp = half_log_2pi * (float)A;
#pragma unroll
    for (int k = 0; k < kAcMaxA; ++k) {
      if (k >= A) break;
      const float ls = a.h.logstd[k];
      const float act = mu[k] + expf(ls) * z[k];
      nlp += 0.5f * z[k] * z[k] + ls;
      if (a.mode == 0) a.r_act[((size_t)a.t * a.rows + r) * A + k] = act;
      a.out[(size_t)r * A + k] = act;
    }
    if (a.mode == 0) {
      a.r_val[(size_t)a.t * a.rows + r] = v;
      a.r_nlp[(size_t)a.t * a.rows + r] = nlp;
    } else {
      if (a.vout) a.vout[r] = v;
      if (a.nlpout) a.nlpout[r] = nlp;
    }
  }
  __syncthreads();
  if (draw && threadIdx.x == 0) *a.step += 1;
}

__global__ void ppo_gae_kernel(const float* __restrict__ rew, const float* __restrict__ val, const float* __restrict__ done,
                               const float* __restrict__ lastv, int T, int E, float gamma, float lam, float* __restrict__ adv,
                               float* __restrict__ ret) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  float last = 0.f;
  for (int t = T - 1; t >= 0; --t) {
    const size_t i = (size_t)t * E + e;
    const float nnt = 1.f - done[(size_t)(t + 1) * E + e];
    const float nv = t == T - 1 ? lastv[e] : val[i + E];
    const float delta = rew[i] + gamma * nv * nnt - val[i];
    last = delta + gamma * lam * nnt * last;
    adv[i] = last;
    ret[i] = last + val[i];
  }
}

// rowoff[i] = (first + i) * XS for the actor's rows
__global__ void ac_iota_rows_kernel(int* __restrict__ rowoff, int first, int n, int XS) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) rowoff[i] = (first + i) * XS;
}

// VecNormalize.normalize_obs of n rows [n][D] into rows of stride XS, one thread per destination element: the float64
// subtract, sqrt, divide and clip in numpy's order, then one rounding to fp32 (NaN passes the clip as np.clip passes it).
// mean == nullptr copies.  The pad columns [D, XS) are written 0.
__global__ void __launch_bounds__(256) ac_obs_norm_kernel(const float* __restrict__ x, int n, int D, int XS,
                                                          const double* __restrict__ mean, const double* __restrict__ var,
                                                          double eps, double clip, float* __restrict__ dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n * XS) return;
  const int r = (int)(i / XS), j = (int)(i - (long long)r * XS);
  float out = 0.f;
  if (j < D) {
    const float v = x[(size_t)r * D + j];
    if (mean) {
      double y = __ddiv_rn(__dsub_rn((double)v, mean[j]), __dsqrt_rn(__dadd_rn(var[j], eps)));
      y = y < -clip ? -clip : (y > clip ? clip : y);
      out = __double2float_rn(y);
    } else {
      out = v;
    }
  }
  dst[i] = out;
}

}  // namespace

int ac_check_net(int obs_dim, int n_actions, int hidden0, int hidden1) {
  if (obs_dim < 1 || obs_dim > 65536) return b2g_fail(B2G_EINVAL, "obs_dim must be in [1, 65536]");
  if (n_actions < 1 || n_actions > kAcMaxA) return b2g_fail(B2G_EINVAL, "n_actions must be in [1, 16]");
  if (hidden0 % 4 || hidden1 % 4 || hidden0 < 4 || hidden1 < 4 || hidden0 > kAcMaxWidth || hidden1 > kAcMaxWidth)
    return b2g_fail(B2G_EINVAL, "hidden widths must be multiples of 4 in [4, 256]");
  return 0;
}

int ac_init(ActorCritic* h, int device, int D, int A, int H0, int H1, int E, int T, int p_rows, uint64_t seed) {
  h->device = device;
  h->D = D; h->XS = (int)ac_row_stride(D); h->A = A; h->H0 = H0; h->H1 = H1;
  h->E = E; h->T = T; h->P_ROWS = p_rows;
  h->act_key = seed ^ 0xA5A5A5A5DEADBEEFull;       // oracle/philox_ref.py act_seed
  h->cfg.device = device;
  h->stage_rows = E;
  h->rms.E = D;
  const char* ng = getenv("B2G_NO_GRAPH");
  h->use_graph = !(ng && ng[0] == '1');
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) return b2g_fail(B2G_ECUDA, "stream");
  return 0;
}

void ac_layout(ActorCritic* h, const std::string& scope, uint32_t grad_mask, int copies) {
  const int64_t D = h->D, A = h->A, H0 = h->H0, H1 = h->H1;
  int64_t off = 0;
  h->oW0 = arena_take(off, D * 2 * H0); h->ob0 = arena_take(off, 2 * H0);
  for (int tw = 0; tw < 2; ++tw) { h->oW1[tw] = arena_take(off, H0 * H1); h->ob1[tw] = arena_take(off, H1); }
  h->oWvf = arena_take(off, H1); h->obvf = arena_take(off, 1); h->oWpi = arena_take(off, H1 * A); h->obpi = arena_take(off, A); h->ols = arena_take(off, A);
  h->n_train = off;
  const int64_t oWq = arena_take(off, H1 * A), obq = arena_take(off, A);
  h->n_total = off;
  h->n_param = copies * h->n_total;
  // zip order (oracle/ppo_ref.py param_specs)
  const struct { const char* name; int64_t rows, cols, stride, off; int ndim; } e[15] = {
      {"pi_fc0/w", D, H0, 2 * H0, h->oW0, 2},     {"pi_fc0/b", 1, H0, H0, h->ob0, 1},
      {"vf_fc0/w", D, H0, 2 * H0, h->oW0 + H0, 2}, {"vf_fc0/b", 1, H0, H0, h->ob0 + H0, 1},
      {"pi_fc1/w", H0, H1, H1, h->oW1[0], 2},     {"pi_fc1/b", 1, H1, H1, h->ob1[0], 1},
      {"vf_fc1/w", H0, H1, H1, h->oW1[1], 2},     {"vf_fc1/b", 1, H1, H1, h->ob1[1], 1},
      {"vf/w", H1, 1, 1, h->oWvf, 2},             {"vf/b", 1, 1, 1, h->obvf, 1},
      {"pi/w", H1, A, A, h->oWpi, 2},             {"pi/b", 1, A, A, h->obpi, 1},
      {"pi/logstd", 1, A, A, h->ols, 2},
      {"q/w", H1, A, A, oWq, 2},                  {"q/b", 1, A, A, obq, 1}};
  for (int i = 0; i < 15; ++i)
    h->params.add(scope + e[i].name, e[i].rows, e[i].cols, e[i].ndim, (int)e[i].stride, e[i].off, (grad_mask >> i) & 1u);
}

int ac_alloc(ActorCritic* h, int rows, AcTab& tab) {
  const int64_t E = h->E, T = h->T, XS = h->XS, A = h->A, H0 = h->H0, H1 = h->H1, R = rows;
  int rc = 0;
#define DA(ptr, count) if ((rc = dev_alloc(h->allocs, h->stream, &(ptr), (size_t)(count)))) return rc
  DA(h->P, h->n_param); DA(h->Mo, h->n_train); DA(h->Vo, h->n_train); DA(h->G, h->n_train);
  DA(h->r_obs, (T + 1) * E * XS); DA(h->r_act, (T + 1) * E * A); DA(h->r_val, (T + 1) * E); DA(h->r_nlp, (T + 1) * E); DA(h->r_rew, T * E);
  DA(h->r_done, (T + 1) * E); DA(h->r_adv, T * E); DA(h->r_ret, T * E); DA(h->lastv, E);
  DA(h->p_obs, (int64_t)h->P_ROWS * XS); DA(h->act_rowoff, E);
  DA(h->Z0, R * 2 * H0); DA(h->Y0, R * 2 * H0); DA(h->Y1, R * 2 * H1);
  DA(h->a_out, R * A); DA(h->a_v, R); DA(h->a_nlp, R);
  DA(h->counters, 4);
#undef DA
  if (cudaMallocHost((void**)&h->h_buf, kAcHostFloats * sizeof(float)) != cudaSuccess) return b2g_fail(B2G_ECUDA, "cudaMallocHost");
  auto up = [&](const char* nm, const std::vector<int>& v) {
    const int* p = nullptr;
    if (int r2 = upload_table(h->allocs, h->stream, v, &p)) return r2;
    tab[nm] = p;
    return 0;
  };
  const int D = h->D;
  if ((rc = up("iD", iota_tab(D))) || (rc = up("iH0", iota_tab((int)H0))) || (rc = up("iH1", iota_tab((int)H1))) ||
      (rc = up("i2H0", iota_tab(2 * (int)H0))) || (rc = up("rM_2H0", iota_tab(rows, 2 * (int)H0))) ||
      (rc = up("rM_2H1", iota_tab(rows, 2 * (int)H1))) || (rc = up("iH0_H1", iota_tab((int)H0, (int)H1))) ||
      (rc = up("iD_2H0", iota_tab(D, 2 * (int)H0))) || (rc = up("boot", iota_tab((int)E, (int)XS, (int)(T * E * XS)))) ||
      (rc = up("pred", iota_tab(h->P_ROWS, (int)XS))))
    return rc;
  if ((rc = ac_make_fwd(h, h->f_act, h->r_obs, h->act_rowoff, (int)E, tab))) return rc;
  if ((rc = ac_make_fwd(h, h->f_boot, h->r_obs, tab["boot"], (int)E, tab))) return rc;
  return ac_make_fwd(h, h->f_pred, h->p_obs, tab["pred"], h->P_ROWS, tab);
}

void ac_release(ActorCritic* h) {
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->graph_exec) cudaGraphExecDestroy(h->graph_exec);
  enc_stage_destroy(h->rms.enc);
  for (void* q : h->allocs) cudaFree(q);
  if (h->h_buf) cudaFreeHost(h->h_buf);
  if (h->stream) cudaStreamDestroy(h->stream);
}

int ac_splits_for(int tiles, int R) {
  const int want = (264 + tiles - 1) / tiles;
  return std::max(1, std::min(want, (R + 63) / 64));
}

int ac_make_fwd(ActorCritic* h, AcFwd& f, const float* obs, const int* rowoff, int M, AcTab& tab) {
  const int D = h->D, H0 = h->H0, H1 = h->H1;
  f.M = M;
  f.l0 = GemmGroup(); f.l1 = GemmGroup();
  f.l0.name = "ppo_l0_fwd"; f.l1.name = "ppo_l1_fwd";
  const int tiles = ((M + 63) / 64) * ((2 * H0 + 63) / 64);
  GemmDesc d = gemm_desc(obs, rowoff, tab["iD"], h->P + h->oW0, tab["iD_2H0"], tab["i2H0"], h->Z0, tab["rM_2H0"], tab["i2H0"], M, 2 * H0, D,
                         GG_A_RVEC | GG_EPI_ATOMIC, ac_splits_for(tiles, D));
  f.l0.host.push_back(d);
  for (int tw = 0; tw < 2; ++tw) {
    GemmDesc g = gemm_desc(h->Y0 + tw * H0, tab["rM_2H0"], tab["iH0"], h->P + h->oW1[tw], tab["iH0_H1"], tab["iH1"], h->Y1 + tw * H1,
                           tab["rM_2H1"], tab["iH1"], M, H1, H0, GG_A_RVEC | GG_EPI_BIAS_TANH);
    g.bias = h->P + h->ob1[tw];
    f.l1.host.push_back(g);
  }
  if (int rc = finalize_tiles(f.l0, h->allocs, h->stream)) return rc;
  return finalize_tiles(f.l1, h->allocs, h->stream);
}

void ac_fwd_issue(ActorCritic* h, const AcFwd& f, cudaStream_t s) {
  cudaMemsetAsync(h->Z0, 0, (size_t)f.M * 2 * h->H0 * sizeof(float), s);
  gg_simt_launch(f.l0.dev, (int)f.l0.host.size(), f.l0.total_tiles, s);
  ac_bias_tanh(h->Z0, h->P + h->ob0, h->Y0, f.M, 2 * h->H0, s);
  gg_simt_launch_tanh(f.l1.dev, (int)f.l1.host.size(), f.l1.total_tiles, s);
}

void ac_bias_tanh(const float* Z, const float* b, float* Y, int n, int N, cudaStream_t s) {
  const int total = n * N;
  ppo_bias_tanh_kernel<<<(total + 255) / 256, 256, 0, s>>>(Z, b, Y, n, N);
}

AcHeadArgs ac_head_args(const ActorCritic* h) {
  AcHeadArgs a{};
  a.Y1 = h->Y1; a.h1 = h->H1; a.A = h->A;
  a.Wpi = h->P + h->oWpi; a.bpi = h->P + h->obpi; a.Wvf = h->P + h->oWvf; a.bvf = h->P + h->obvf; a.logstd = h->P + h->ols;
  return a;
}

AcActArgs ac_act_args(ActorCritic* h, int rows, int mode) {
  AcActArgs a{};
  a.h = ac_head_args(h); a.rows = rows; a.mode = mode; a.key = h->act_key; a.step = h->counters + 1;
  a.r_act = h->r_act; a.r_val = h->r_val; a.r_nlp = h->r_nlp; a.lastv = h->lastv;
  a.out = h->a_out; a.vout = h->a_v; a.nlpout = h->a_nlp;
  return a;
}

void ac_act(const AcActArgs& a, cudaStream_t s) { ppo_act_kernel<<<1, kAcActThreads, 0, s>>>(a); }

void ac_gae(const float* rew, const float* val, const float* done, const float* lastv, int T, int E, float gamma, float lam, float* adv,
            float* ret, cudaStream_t s) {
  ppo_gae_kernel<<<(E + 127) / 128, 128, 0, s>>>(rew, val, done, lastv, T, E, gamma, lam, adv, ret);
}

int ac_upload_rows(ActorCritic* h, float* dst, const float* src, int rows) {
  CK(cudaMemcpy2DAsync(dst, h->XS * sizeof(float), src, h->D * sizeof(float), h->D * sizeof(float), rows, cudaMemcpyDefault, h->stream));
  return 0;
}

namespace {

// the forward pass and the stream-1 draw of rollout row t (its observations in place) -> act_out, enqueued
int act_row(ActorCritic* h, float* act_out) {
  cudaStream_t s = h->stream;
  ac_iota_rows_kernel<<<(h->E + 255) / 256, 256, 0, s>>>(h->act_rowoff, h->t * h->E, h->E, h->XS);
  ac_fwd_issue(h, h->f_act, s);
  AcActArgs a = ac_act_args(h, h->E, 0);
  a.t = h->t;
  ac_act(a, s);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(act_out, h->a_out, (size_t)h->E * h->A * sizeof(float), cudaMemcpyDefault, s));
  h->acted = true;
  return 0;
}

int ensure_stage(ActorCritic* h) {
  if (h->ob_stage) return 0;
  return dev_alloc(h->allocs, h->stream, &h->ob_stage, (size_t)std::max(h->E, h->P_ROWS) * h->D);
}

}  // namespace

int ac_rollout_act(ActorCritic* h, const float* obs, float* act_out) {
  CK(cudaSetDevice(h->device));
  if (int rc = ac_upload_rows(h, h->r_obs + (size_t)h->t * h->E * h->XS, obs, h->E)) return rc;
  h->ob_n = 0;
  if (int rc = act_row(h, act_out)) return rc;
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}

int ac_rollout_reward(ActorCritic* h, const float* rew, const float* done) {
  CK(cudaSetDevice(h->device));
  const size_t E = h->E;
  CK(cudaMemcpyAsync(h->r_rew + (size_t)h->t * E, rew, E * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaMemcpyAsync(h->r_done + (size_t)(h->t + 1) * E, done, E * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaStreamSynchronize(h->stream));      // rew and done may live on the caller's stack
  h->t += 1;
  h->acted = false;
  return 0;
}

int ac_rollout_reset(ActorCritic* h) {
  CK(cudaSetDevice(h->device));
  CK(cudaMemsetAsync(h->r_done, 0, (size_t)h->E * sizeof(float), h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->t = 0;
  h->acted = false;
  h->ob_n = 0;
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------
// obs_rms on the device and the observe path
// ---------------------------------------------------------------------------------------------------------------------------
void ac_obs_normalize(const ActorCritic* h, const float* x, int n, float* dst, cudaStream_t s) {
  const bool norm = h->rms.on() && h->norm_obs;
  const long long total = (long long)n * h->XS;
  ac_obs_norm_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(x, n, h->D, h->XS, norm ? h->rms.mean : nullptr,
                                                                     norm ? h->rms.var : nullptr, h->rms.eps, h->clip_obs, dst);
}

int ac_obs_rms_set(ActorCritic* h, const double* mean, const double* var, double count) {
  if (h && !h->rms_tab) {      // ObsRms::merge rewrites a table as it merges; allocated with obs_rms
    CK(cudaSetDevice(h->device));
    if (int rc = dev_alloc(h->allocs, h->stream, &h->rms_tab, 2 * (size_t)h->D)) return rc;
    h->rms.d_mean = h->rms_tab;
    h->rms.d_istd = h->rms_tab + h->D;
  }
  return obs_rms_set(h, mean, var, count);
}

int ac_obs_rms_get(ActorCritic* h, double* mean, double* var, double* count) { return obs_rms_get(h, mean, var, count); }

int ac_upload_bytes(const ActorCritic* h, int64_t* observe_bytes, int64_t* other_bytes) {
  return obs_rms_upload_bytes(h, observe_bytes, other_bytes);
}

int ac_set_norm_stats(ActorCritic* h, double clip_obs, double eps, int norm_obs) {
  if (!(clip_obs >= 0.0) || !std::isfinite(clip_obs) || !(eps >= 0.0) || !std::isfinite(eps))
    return b2g_fail(B2G_EINVAL, "set_norm_stats: clip_obs and epsilon must be finite and >= 0");
  CK(cudaSetDevice(h->device));
  if (int rc = h->rms.norm_stats(nullptr, nullptr, eps, h->cfg.device, h->cfg.nranks, h->allocs, h->stream)) return rc;
  h->clip_obs = clip_obs;      // a kernel argument: observe calls enqueued later read the new value
  h->norm_obs = norm_obs != 0;
  return 0;
}

int ac_set_obs_encoder(ActorCritic* h, const b2g_encoder* enc, int tail) {
  if (enc)
    if (int rc = obs_rms_check_encoder(h, enc, tail)) return rc;
  return obs_rms_attach_encoder(h, enc, tail);
}

int ac_observe_act(ActorCritic* h, const float* obs, int n, int update_stats, float* act_out, bool carried) {
  if (!obs && !act_out) return b2g_fail(B2G_EINVAL, "observe_act: nothing to do (obs and act_out are NULL)");
  if (n != h->E) return b2g_fail(B2G_EINVAL, "observe_act: n must be the handle's n_envs (" + std::to_string(h->E) + ")");
  if (obs && update_stats && !h->rms.on())
    return b2g_fail(B2G_ESTATE, std::string("update_stats needs device statistics: call ") + h->rms.set_call + " first");
  const int row = h->t + (h->acted ? 1 : 0);     // the row an observation staged now belongs to
  if (act_out) {
    if (h->t >= h->T) return b2g_fail(B2G_ESTATE, "observe_act: the rollout is full: update first");
    if (h->acted) return b2g_fail(B2G_ESTATE, "observe_act: row t's action is drawn: pass its rewards (rollout_reward) first");
    if (!obs && !(h->ob_n && h->ob_row == h->t))
      return b2g_fail(B2G_ESTATE, "observe_act: no observation staged in the current row (pass obs first)");
  } else if (row > h->T) {
    return b2g_fail(B2G_ESTATE, "observe_act: the rollout is full: update first");
  }
  CK(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  if (obs) {
    if (int rc = ensure_stage(h)) return rc;
    if (int rc = h->rms.stage_frames(h->ob_stage, obs, n, s)) return rc;
    if (update_stats) h->rms.merge(h->ob_stage, nullptr, nullptr, n, s);
    ac_obs_normalize(h, h->ob_stage, n, h->r_obs + (size_t)row * h->E * h->XS, s);
    h->ob_n = n;
    h->ob_row = row;
  }
  if (act_out) {
    if (carried && h->t == 0) {      // the action drawn for this row before the last update
      CK(cudaMemcpyAsync(act_out, h->r_act, (size_t)h->E * h->A * sizeof(float), cudaMemcpyDefault, s));
      h->acted = true;
    } else if (int rc = act_row(h, act_out)) {
      return rc;
    }
  }
  CK(cudaStreamSynchronize(s));      // caller-owned arrays are copied, the actions are the result of the call
  CK(cudaGetLastError());
  return 0;
}

int ac_check_last_obs(const ActorCritic* h, const float* last_obs) {
  if (last_obs || (h->ob_n && h->ob_row == h->T)) return 0;
  return b2g_fail(B2G_EINVAL, "update: last_obs is NULL and no observation is staged in the bootstrap row (observe_act after the "
                              "last step)");
}

int ac_update_last_obs(ActorCritic* h, const float* last_obs) {
  if (!last_obs) return 0;
  h->ob_n = 0;
  return ac_upload_rows(h, h->r_obs + (size_t)h->T * h->E * h->XS, last_obs, h->E);
}

int ac_update_finish(ActorCritic* h, const float* last_obs, bool copy_row0) {
  h->acted = false;
  if (last_obs) return 0;
  if (copy_row0)
    CK(cudaMemcpyAsync(h->r_obs, h->r_obs + (size_t)h->T * h->E * h->XS, (size_t)h->E * h->XS * sizeof(float), cudaMemcpyDeviceToDevice,
                       h->stream));
  h->ob_row = 0;
  return 0;
}

int ac_rollout_get(ActorCritic* h, float* adv, float* ret, float* val, float* nlp, float* act) {
  CK(cudaSetDevice(h->device));
  CK(cudaStreamSynchronize(h->stream));
  const size_t n = (size_t)h->T * h->E;
  if (adv) CK(cudaMemcpy(adv, h->r_adv, n * sizeof(float), cudaMemcpyDeviceToHost));
  if (ret) CK(cudaMemcpy(ret, h->r_ret, n * sizeof(float), cudaMemcpyDeviceToHost));
  if (val) CK(cudaMemcpy(val, h->r_val, n * sizeof(float), cudaMemcpyDeviceToHost));
  if (nlp) CK(cudaMemcpy(nlp, h->r_nlp, n * sizeof(float), cudaMemcpyDeviceToHost));
  if (act) CK(cudaMemcpy(act, h->r_act, n * h->A * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

int ac_run_update(ActorCritic* h, const std::function<int()>& issue) {
  if (h->use_graph && !h->graph_exec)
    if (int rc = capture_graph(h->stream, issue, &h->graph_exec)) return rc;
  if (h->graph_exec) CK(cudaGraphLaunch(h->graph_exec, h->stream));
  else if (int rc = issue()) return rc;
  return 0;
}

int ac_predict(ActorCritic* h, const float* obs, int n, int deterministic, float* act_out, float* value_out, float* nlp_out, bool raw) {
  CK(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const int P = h->P_ROWS;
  if (raw)
    if (int rc = ensure_stage(h)) return rc;
  for (int done_n = 0; done_n < n; done_n += P) {
    const int chunk = std::min(P, n - done_n);
    if (raw) {
      const size_t bytes = (size_t)chunk * h->D * sizeof(float);
      CK(cudaMemcpyAsync(h->ob_stage, obs + (size_t)done_n * h->D, bytes, cudaMemcpyDefault, s));
      h->rms.up_other += (int64_t)bytes;
      ac_obs_normalize(h, h->ob_stage, chunk, h->p_obs, s);
    } else if (int rc = ac_upload_rows(h, h->p_obs, obs + (size_t)done_n * h->D, chunk)) {
      return rc;
    }
    ac_fwd_issue(h, h->f_pred, s);
    AcActArgs a = ac_act_args(h, chunk, 2);
    a.deterministic = deterministic;
    ac_act(a, s);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(act_out + (size_t)done_n * h->A, h->a_out, (size_t)chunk * h->A * sizeof(float), cudaMemcpyDefault, s));
    if (value_out) CK(cudaMemcpyAsync(value_out + done_n, h->a_v, chunk * sizeof(float), cudaMemcpyDefault, s));
    if (nlp_out) CK(cudaMemcpyAsync(nlp_out + done_n, h->a_nlp, chunk * sizeof(float), cudaMemcpyDefault, s));
    CK(cudaStreamSynchronize(s));
  }
  return 0;
}

int ac_get_step(ActorCritic* h, int64_t* adam_step, int64_t* noise_step, int32_t* rollout_rows) {
  CK(cudaSetDevice(h->device));
  CK(cudaStreamSynchronize(h->stream));
  long long c[2];
  CK(cudaMemcpy(c, h->counters, sizeof c, cudaMemcpyDeviceToHost));
  if (adam_step) *adam_step = c[0];
  if (noise_step) *noise_step = c[1];
  if (rollout_rows) *rollout_rows = h->t;
  return 0;
}

bool ac_debug_base(const ActorCritic* h, int rows, const std::string& name, AcDebugBuf& b) {
  const int64_t E = h->E, T = h->T, A = h->A, R = rows;
  const struct { const char* nm; const void* p; int64_t n; int eb; } t[] = {
      {"P", h->P, h->n_param, 4},          {"G", h->G, h->n_train, 4},           {"Mo", h->Mo, h->n_train, 4},
      {"Vo", h->Vo, h->n_train, 4},        {"Z0", h->Z0, R * 2 * h->H0, 4},      {"Y0", h->Y0, R * 2 * h->H0, 4},
      {"Y1", h->Y1, R * 2 * h->H1, 4},     {"r_obs", h->r_obs, (T + 1) * E * h->XS, 4}, {"r_act", h->r_act, (T + 1) * E * A, 4},
      {"r_val", h->r_val, (T + 1) * E, 4}, {"r_nlp", h->r_nlp, (T + 1) * E, 4},  {"r_rew", h->r_rew, T * E, 4},
      {"r_done", h->r_done, (T + 1) * E, 4}, {"r_adv", h->r_adv, T * E, 4},      {"r_ret", h->r_ret, T * E, 4},
      {"lastv", h->lastv, E, 4},           {"a_out", h->a_out, R * A, 4},        {"a_v", h->a_v, R, 4},
      {"a_nlp", h->a_nlp, R, 4},           {"act_rowoff", h->act_rowoff, E, 4},  {"counters", h->counters, 4, 8}};
  for (const auto& e : t)
    if (name == e.nm) { b.p = e.p; b.numel = e.n; b.elem_bytes = e.eb; return true; }
  return false;
}

int ac_debug_info(const AcDebugBuf& b, int64_t* numel, int32_t* elem_bytes) {
  if (numel) *numel = b.numel;
  if (elem_bytes) *elem_bytes = b.elem_bytes;
  return 0;
}

int ac_debug_read(ActorCritic* h, const AcDebugBuf& b, const char* name, void* dst, size_t bytes) {
  if (bytes != (size_t)b.numel * b.elem_bytes) return b2g_fail(B2G_EINVAL, std::string(name) + ": size mismatch");
  CK(cudaSetDevice(h->device));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaMemcpy(dst, b.p, bytes, cudaMemcpyDeviceToHost));
  return 0;
}

namespace {
// sections 2..: the parameter arena and the Adam moments, then obs_rms when the handle owns it
std::vector<StateSection> ac_device_sections(ActorCritic* h) {
  std::vector<StateSection> s = adam_sections(h->P, h->n_param, h->Mo, h->Vo, h->n_train);
  if (h->rms.on()) s.push_back(rms_section(&h->rms.count, h->rms.mean, h->rms.var, h->D));
  return s;
}
}  // namespace

int ac_state_save(ActorCritic* h, const char* path, uint32_t kind, const std::vector<FpField>& fp) {
  CK(cudaSetDevice(h->device));
  CK(cudaStreamSynchronize(h->stream));
  long long cnt[4];
  CK(cudaMemcpy(cnt, h->counters, sizeof cnt, cudaMemcpyDeviceToHost));
  int64_t hv[2] = {h->n_updates, 0};
  std::vector<StateSection> secs = host_sections(hv, sizeof hv, cnt, sizeof cnt);
  for (auto& s : ac_device_sections(h)) secs.push_back(std::move(s));
  return state_write(path, kind, fp_with_rms(fp, h->rms.on()), secs);
}

int ac_state_load(ActorCritic* h, const char* path, uint32_t kind, const std::vector<FpField>& fp, const char* learner) {
  CK(cudaSetDevice(h->device));
  StateReader rd;
  if (int rc = state_open_rms(rd, path, kind, fp, h->rms.on(), h->rms.set_call)) return rc;
  const std::vector<StateSection> dev = ac_device_sections(h);
  if (int rc = state_check_tags(rd, dev, learner)) return rc;
  int64_t hv[2];
  long long cnt[4];
  if (rd.bytes(0) != sizeof hv || rd.bytes(1) != sizeof cnt)
    return b2g_fail(B2G_EINVAL, "training-state section lengths do not match this handle's configuration");
  if (int rc = state_check_lengths(rd, dev)) return rc;
  if (int rc = rd.read_host(0, hv, sizeof hv)) return rc;
  if (int rc = rd.read_host(1, cnt, sizeof cnt)) return rc;
  CK(cudaStreamSynchronize(h->stream));
  return state_read_device(rd, dev, &h->broken, [&] {
    CK(cudaMemcpy(h->counters, cnt, sizeof cnt, cudaMemcpyHostToDevice));
    CK(cudaMemset(h->r_done, 0, (size_t)h->E * sizeof(float)));
    if (h->rms.on()) {      // the table ObsRms keeps beside obs_rms
      h->rms.derive(h->stream);
      CK(cudaStreamSynchronize(h->stream));
    }
    h->n_updates = hv[0];
    h->t = 0;
    h->acted = false;
    h->ob_n = 0;
    return 0;
  });
}

}  // namespace b2g
