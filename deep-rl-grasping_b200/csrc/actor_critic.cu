// The actor-critic MLP and rollout kernels the PPO2 and TRPO handles share (actor_critic.cuh).
#include <cuda_runtime.h>
#include <math.h>

#include <algorithm>

#include "actor_critic.cuh"
#include "host.cuh"

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

}  // namespace

int ac_splits_for(int tiles, int R) {
  const int want = (264 + tiles - 1) / tiles;
  return std::max(1, std::min(want, (R + 63) / 64));
}

int ac_make_fwd(ActorCritic* h, AcFwd& f, const float* obs, const int* rowoff, int M, std::map<std::string, const int*>& tab) {
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

}  // namespace b2g
