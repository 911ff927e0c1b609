// libb200grasp: TRPO learner -- the `sb.TRPO` branch of sb_helper.py:129-136 (stable-baselines 2.10.1 trpo_mpi, one env,
// restated in tests/trpo_ref.py).
//
// Network: PPO2's MlpPolicy (actor_critic.cuh), live under pi/model/ and copied under oldpi/model/ (the old policy: a second
// copy of the whole block behind the first in the parameter arena).
//
// Update (b2g_trpo_update, one CUDA graph; the only host synchronise reads the metrics):
//   boundary  forward of the boundary observation with the old parameters: its stream-1 action (row 0 of the next batch) and
//             the bootstrap value; GAE over the N rows
//   oldpi     oldpi := pi
//   gradient  forward at theta_old over the batch, trpo_prep_kernel (atarg, mean / logp at theta_old, the losses, the seeds),
//             the pi tower's backward on gg_simt, trpo_headgrad_kernel (pi/w, pi/b, logstd)
//   CG        cg_iters iterations of z = F p (forward-mode tangent through the pi tower over the rows [::5], then its backward:
//             F = J^T diag(1 / (sigma^2 N_f)) J for the mean, 2 I for logstd, + damping), fixed-order double dot products and
//             device scalars: once r.r < 1e-10 the remaining iterations' vector updates are no-ops
//   step      shs = 0.5 x.Fx, fullstep = x / sqrt(|shs| / max_kl), expectedimprove = g.fullstep
//   search    the ten candidates 0.5^k share layer 0: Z0 + s_k (X dW0) needs one extra D-deep contraction; layer 1 of the ten is
//             one grouped launch; the losses of all ten in one kernel; the select kernel applies the first acceptable k
//   value     vf_iters passes of N / 128 minibatches in the caller's permutation: vf tower forward, loss mean (V - R)^2, its
//             backward and MpiAdam (epsilon 1e-8, no clipping)
//   carry     row 0 of the next batch: the boundary observation and action, its value under the updated value tower
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

constexpr int kMaxN = 16384;         // timesteps_per_batch: one CTA standardises the advantages
constexpr int kPrepThreads = 1024;
constexpr int kDotBlocks = 128, kDotThreads = 256;
constexpr int kLsBlocks = 64, kLsThreads = 256;
constexpr int kNcand = 10;           // line-search step sizes 0.5^k, k = 0..9
constexpr int kVfBatch = 128;        // value minibatch rows
constexpr float kAdamEps = 1e-8f;    // common/mpi_adam.py
constexpr double kHalfLog2Pi = 0.91893853320467274, kHalfLog2PiE = 1.4189385332046727;

// metric slots (float): losses before [0, 5), after [5, 10), then the scalars
enum : int { TM_BEFORE = 0, TM_AFTER = 5, TM_GG = 10, TM_SHS, TM_EI, TM_VF, TM_N = 16 };
// device scalars (double)
enum : int { SC_RR = 0, SC_ALPHA, SC_BETA, SC_DONE, SC_ZERO, SC_BAD, SC_ITERS, SC_ACC, SC_LM, SC_N = 16 };

// the value minibatches' storage rows: rowoff[i] = perm[i] * XS
__global__ void trpo_rows_kernel(const int* __restrict__ perm, int n, int XS, int* __restrict__ rowoff) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) rowoff[i] = perm[i] * XS;
}

struct PrepArgs {
  AcHeadArgs h;                      // theta_old forward over the batch
  int N;
  const float* act; const float* adv;
  float entcoeff;
  float* atarg; float* mu_old; float* nlp_old;   // [N], [N, A], [N]
  float* sdm; float* sdls;                       // gradient seeds d optimgain / d mu, d / d logstd per row [N, A]
  float* met;
};

// atarg = (adv - mean) / (std + 1e-8) (population std), the losses at theta_old and the per-row gradient seeds
__global__ void __launch_bounds__(kPrepThreads) trpo_prep_kernel(PrepArgs a) {
  __shared__ double red[kPrepThreads / 32];
  const int N = a.N, A = a.h.A, tid = threadIdx.x, NT = blockDim.x;
  double s = 0.0;
  for (int r = tid; r < N; r += NT) s += (double)a.adv[r];
  const double mean = block_sum_t(s, red) / N;
  double ss = 0.0;
  for (int r = tid; r < N; r += NT) { const double d = (double)a.adv[r] - mean; ss += d * d; }
  const double stdv = sqrt(block_sum_t(ss, red) / N);
  const float invN = 1.0f / (float)N;
  double sg = 0.0;
  for (int r = tid; r < N; r += NT) {
    const float at = (float)(((double)a.adv[r] - mean) / (stdv + 1e-8));
    a.atarg[r] = at;
    sg += (double)at;
    float mu[kAcMaxA], v;
    ac_heads(a.h, r, mu, v);
    float nlp = (float)kHalfLog2Pi * (float)A;
#pragma unroll
    for (int k = 0; k < kAcMaxA; ++k) {
      if (k >= A) break;
      const float ls = a.h.logstd[k], sig = expf(ls);
      const float d = a.act[(size_t)r * A + k] - mu[k];
      const float z = d / sig;
      nlp += 0.5f * z * z + ls;
      a.mu_old[(size_t)r * A + k] = mu[k];
      a.sdm[(size_t)r * A + k] = at * z / sig * invN;              // d/dmu of ratio * atarg at ratio = 1
      a.sdls[(size_t)r * A + k] = at * (z * z - 1.f) * invN;        // d/dlogstd
    }
    a.nlp_old[r] = nlp;
  }
  const double surr = block_sum_t(sg, red) / N;     // ratio = exp(0) = 1 at theta_old
  if (tid == 0) {
    double ent = kHalfLog2PiE * A;
    for (int k = 0; k < A; ++k) ent += (double)a.h.logstd[k];
    const double eb = (double)a.entcoeff * ent;
    const float m[5] = {(float)(surr + eb), 0.f, (float)eb, (float)surr, (float)ent};
    for (int k = 0; k < 5; ++k) { a.met[TM_BEFORE + k] = m[k]; a.met[TM_AFTER + k] = m[k]; }
  }
}

// dZ1[r, k] = (sum_j seed[r, j] Wpi[k, j]) (1 - y^2), y = Y1[r * ys + k]: the head's backward into the pi tower (compact rows)
__global__ void trpo_head_bwd_kernel(const float* __restrict__ seed, const float* __restrict__ Wpi, const float* __restrict__ Y1, int ys,
                                     int M, int h1, int A, float* __restrict__ dZ1) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * h1) return;
  const int r = i / h1, k = i - r * h1;
  const float* sd = seed + (size_t)r * A;
  const float* w = Wpi + (size_t)k * A;
  float d = 0.f;
  for (int j = 0; j < A; ++j) d = fmaf(sd[j], w[j], d);
  const float y = Y1[(size_t)r * ys + k];
  dZ1[i] = d * (1.f - y * y);
}

// one output per CTA, summed over the M rows in double (fixed order): gWpi[k, j] = sum_r Y1[r, k] seed[r, j], gbpi[j] =
// sum_r seed[r, j] and, with sls, glogstd[j] = sum_r sls[r, j] + entcoeff
__global__ void __launch_bounds__(256) trpo_headgrad_kernel(const float* __restrict__ Y1, int ys, const float* __restrict__ seed,
                                                            const float* __restrict__ sls, float entcoeff, int M, int h1, int A,
                                                            float* gWpi, float* gbpi, float* gls) {
  __shared__ double red[8];
  const int jb = blockIdx.x, nW = h1 * A;
  double s = 0.0;
  if (jb < nW) {
    const int k = jb / A, j = jb - k * A;
    for (int r = threadIdx.x; r < M; r += blockDim.x) s += (double)Y1[(size_t)r * ys + k] * (double)seed[(size_t)r * A + j];
  } else if (jb < nW + A) {
    const int j = jb - nW;
    for (int r = threadIdx.x; r < M; r += blockDim.x) s += (double)seed[(size_t)r * A + j];
  } else {
    const int j = jb - nW - A;
    for (int r = threadIdx.x; r < M; r += blockDim.x) s += (double)sls[(size_t)r * A + j];
  }
  const double t = block_sum_t(s, red);
  if (threadIdx.x == 0) {
    if (jb < nW) gWpi[jb] = (float)t;
    else if (jb < nW + A) gbpi[jb - nW] = (float)t;
    else gls[jb - nW - A] = (float)(t + entcoeff);
  }
}

// tangent of a tanh layer: T[r, c] = (1 - y^2) (T[r, c] + vb[c]), y = Y[r * ys + c]  (T compact [M, H])
__global__ void trpo_tangent_kernel(float* __restrict__ T, const float* __restrict__ vb, const float* __restrict__ Y, int ys, int M, int H) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * H) return;
  const int r = i / H, c = i - r * H;
  const float y = Y[(size_t)r * ys + c];
  T[i] = (1.f - y * y) * (T[i] + vb[c]);
}

// the mean's tangent J v at row r and the Fisher weighting: u[r, j] = (dY1 Wpi + Y1 Vpi + vbpi)_j / (sigma_j^2 M)
__global__ void trpo_fvp_head_kernel(const float* __restrict__ dY1, const float* __restrict__ Y1, int ys, const float* __restrict__ Wpi,
                                     const float* __restrict__ Vpi, const float* __restrict__ vbpi, const float* __restrict__ logstd,
                                     int M, int h1, int A, float* __restrict__ u) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= M) return;
  float d[kAcMaxA];
#pragma unroll
  for (int j = 0; j < kAcMaxA; ++j) d[j] = j < A ? vbpi[j] : 0.f;
  for (int k = 0; k < h1; ++k) {
    const float t = dY1[(size_t)r * h1 + k], y = Y1[(size_t)r * ys + k];
#pragma unroll
    for (int j = 0; j < kAcMaxA; ++j)
      if (j < A) d[j] = fmaf(t, Wpi[(size_t)k * A + j], fmaf(y, Vpi[(size_t)k * A + j], d[j]));
  }
#pragma unroll
  for (int j = 0; j < kAcMaxA; ++j)
    if (j < A) u[(size_t)r * A + j] = d[j] / (expf(2.f * logstd[j]) * (float)M);
}

// z += damping v, and the logstd block's 2 v
__global__ void trpo_fvp_finish_kernel(float* __restrict__ z, const float* __restrict__ v, int n, int64_t ols, int A, float damping) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float t = z[i] + damping * v[i];
  if (i >= ols && i < ols + A) t += 2.f * v[i];
  z[i] = t;
}

// fixed-grid partials of a . b in double, and of max |a| when amax is given
__global__ void __launch_bounds__(kDotThreads) trpo_dot_kernel(const float* __restrict__ a, const float* __restrict__ b, int n,
                                                               double* __restrict__ part, double* __restrict__ amax) {
  __shared__ double red[kDotThreads / 32];
  double s = 0.0, m = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    s += (double)a[i] * (double)b[i];
    m = fmax(m, fabs((double)a[i]));
  }
  const double t = block_sum_t(s, red);
  if (threadIdx.x == 0) part[blockIdx.x] = t;
  if (amax) {
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
      double mm = 0.0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) mm = fmax(mm, red[w]);
      amax[blockIdx.x] = mm;
    }
  }
}

__device__ __forceinline__ double sum_parts(const double* part) {
  double s = 0.0;
  for (int i = 0; i < kDotBlocks; ++i) s += part[i];
  return s;
}

// the scalar steps of conjugate gradient and of the step size (one thread)
enum : int { CG_INIT = 0, CG_ALPHA, CG_BETA, CG_CHECK, CG_SHS, CG_EI };
__global__ void trpo_conjgrad_kernel(int stage, const double* __restrict__ part, const double* __restrict__ amax, double* sc, float* met,
                               float max_kl) {
  if (threadIdx.x != 0) return;
  const double s = sum_parts(part);
  switch (stage) {
    case CG_INIT: {                  // s = g.g; np.allclose(g, 0): every |g_i| <= 1e-8
      double m = 0.0;
      for (int i = 0; i < kDotBlocks; ++i) m = fmax(m, amax[i]);
      sc[SC_RR] = s;
      sc[SC_ZERO] = m <= 1e-8 ? 1.0 : 0.0;
      sc[SC_DONE] = sc[SC_ZERO];
      sc[SC_BAD] = 0.0;
      sc[SC_ITERS] = 0.0;
      sc[SC_ACC] = -2.0;
      met[TM_GG] = (float)s;
      met[TM_SHS] = 0.f; met[TM_EI] = 0.f;
      break;
    }
    case CG_ALPHA:                   // s = p.z
      if (sc[SC_DONE] == 0.0) sc[SC_ALPHA] = sc[SC_RR] / s;
      break;
    case CG_BETA:                    // s = r.r after the update
      if (sc[SC_DONE] == 0.0) {
        sc[SC_BETA] = s / sc[SC_RR];
        sc[SC_RR] = s;
        sc[SC_ITERS] += 1.0;
        if (s < 1e-10) sc[SC_DONE] = 2.0;     // the p update of this iteration still runs (it is not read again)
      }
      break;
    case CG_CHECK:                   // s = x.x: assert np.isfinite(stepdir).all()
      if (sc[SC_ZERO] == 0.0 && !isfinite(s)) sc[SC_BAD] = 1.0;
      break;
    case CG_SHS:                     // s = x.Fx
      if (sc[SC_ZERO] == 0.0 && sc[SC_BAD] == 0.0) {
        const double shs = 0.5 * s;
        sc[SC_LM] = sqrt(fabs(shs) / (double)max_kl);
        met[TM_SHS] = (float)shs;
      }
      break;
    case CG_EI:                      // s = g.fullstep
      if (sc[SC_ZERO] == 0.0 && sc[SC_BAD] == 0.0) met[TM_EI] = (float)s;
      break;
  }
}

// vector steps.  op 0: x = 0, r = p = g;  op 1: x += alpha p, r -= alpha z;  op 2: p = r + beta p;  op 3: fullstep = x / lm (0
// without a policy step)
__global__ void trpo_vec_kernel(int op, int n, const double* __restrict__ sc, const float* __restrict__ g, float* __restrict__ x,
                                float* __restrict__ r, float* __restrict__ p, const float* __restrict__ z, float* __restrict__ fs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (op == 0) { x[i] = 0.f; r[i] = g[i]; p[i] = g[i]; return; }
  if (op == 3) {
    fs[i] = (sc[SC_ZERO] == 0.0 && sc[SC_BAD] == 0.0) ? (float)((double)x[i] / sc[SC_LM]) : 0.f;
    return;
  }
  if (op == 1) {
    if (sc[SC_DONE] != 0.0) return;
    const float al = (float)sc[SC_ALPHA];
    x[i] = fmaf(al, p[i], x[i]);
    r[i] = fmaf(-al, z[i], r[i]);
  } else {
    if (sc[SC_DONE] == 1.0) return;
    p[i] = fmaf((float)sc[SC_BETA], p[i], r[i]);
  }
}

__device__ __forceinline__ float cand_value(float p, float f, float s) { return __fadd_rn(p, __fmul_rn(s, f)); }

struct CandArgs {
  const float* P; const float* fs;
  int64_t ob0, oW1, ob1, oWpi, obpi, ols;
  int H0, H1, A;
  float *b0c, *W1c, *b1c, *Wpic, *bpic, *lsc;   // [kNcand][...]
};

// the pi tower's candidate parameters theta_old + 0.5^k fullstep (layer 0's weights enter through Z0 + s dZ)
__global__ void trpo_cand_kernel(CandArgs a) {
  const int k = blockIdx.y;
  const float s = ldexpf(1.f, -k);
  const int n0 = a.H0, n1 = a.H0 * a.H1, n2 = a.H1, n3 = a.H1 * a.A, n4 = a.A, n5 = a.A;
  const int tot = n0 + n1 + n2 + n3 + n4 + n5;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < tot; i += gridDim.x * blockDim.x) {
    int j = i;
    if (j < n0) { a.b0c[(size_t)k * n0 + j] = cand_value(a.P[a.ob0 + j], a.fs[a.ob0 + j], s); continue; }
    j -= n0;
    if (j < n1) { a.W1c[(size_t)k * n1 + j] = cand_value(a.P[a.oW1 + j], a.fs[a.oW1 + j], s); continue; }
    j -= n1;
    if (j < n2) { a.b1c[(size_t)k * n2 + j] = cand_value(a.P[a.ob1 + j], a.fs[a.ob1 + j], s); continue; }
    j -= n2;
    if (j < n3) { a.Wpic[(size_t)k * n3 + j] = cand_value(a.P[a.oWpi + j], a.fs[a.oWpi + j], s); continue; }
    j -= n3;
    if (j < n4) { a.bpic[(size_t)k * n4 + j] = cand_value(a.P[a.obpi + j], a.fs[a.obpi + j], s); continue; }
    j -= n4;
    a.lsc[(size_t)k * n5 + j] = cand_value(a.P[a.ols + j], a.fs[a.ols + j], s);
  }
}

// layer 0 of candidate k: Y0[k][r, c] = tanh(Z0[r, c] + 0.5^k dZ[r, c] + b0c[k][c])   (Z0: theta_old's X W0, row stride zs)
__global__ void trpo_ls_l0_kernel(const float* __restrict__ Z0, int zs, const float* __restrict__ dZ, const float* __restrict__ b0c,
                                  int N, int H0, float* __restrict__ Y0) {
  const int k = blockIdx.y;
  const float s = ldexpf(1.f, -k);
  const int64_t n = (int64_t)N * H0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / H0), c = (int)(i - (int64_t)r * H0);
    Y0[(size_t)k * n + i] = tanhf(Z0[(size_t)r * zs + c] + s * dZ[i] + b0c[(size_t)k * H0 + c]);
  }
}

struct LsArgs {
  const float* Y1c;                  // [kNcand][N, H1]
  const float *Wpic, *bpic, *lsc;    // [kNcand][...]
  const float *mu_old, *nlp_old, *atarg, *act, *ls_old;
  int N, H1, A;
  double* part;                      // [kNcand][kLsBlocks][2]: surrogate and KL sums
};

// per-row surrogate ratio * atarg and KL(old || new) of every candidate, fixed-order double partials
__global__ void __launch_bounds__(kLsThreads) trpo_ls_loss_kernel(LsArgs a) {
  __shared__ double red[kLsThreads / 32];
  const int k = blockIdx.y, A = a.A, H1 = a.H1;
  const float* Y1 = a.Y1c + (size_t)k * a.N * H1;
  const float* W = a.Wpic + (size_t)k * H1 * A;
  const float* b = a.bpic + (size_t)k * A;
  const float* ls = a.lsc + (size_t)k * A;
  double ss = 0.0, sk = 0.0;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < a.N; r += gridDim.x * blockDim.x) {
    float mu[kAcMaxA];
#pragma unroll
    for (int j = 0; j < kAcMaxA; ++j) mu[j] = j < A ? b[j] : 0.f;
    for (int q = 0; q < H1; ++q) {
      const float y = Y1[(size_t)r * H1 + q];
#pragma unroll
      for (int j = 0; j < kAcMaxA; ++j)
        if (j < A) mu[j] = fmaf(y, W[(size_t)q * A + j], mu[j]);
    }
    float nlp = (float)kHalfLog2Pi * (float)A;
    double kl = 0.0;
#pragma unroll
    for (int j = 0; j < kAcMaxA; ++j) {
      if (j >= A) break;
      const float sig = expf(ls[j]);
      const float z = (a.act[(size_t)r * A + j] - mu[j]) / sig;
      nlp += 0.5f * z * z + ls[j];
      const double so = exp((double)a.ls_old[j]), sn = exp((double)ls[j]);
      const double dm = (double)a.mu_old[(size_t)r * A + j] - (double)mu[j];
      kl += (double)ls[j] - (double)a.ls_old[j] + (so * so + dm * dm) / (2.0 * sn * sn) - 0.5;
    }
    ss += exp((double)a.nlp_old[r] - (double)nlp) * (double)a.atarg[r];
    sk += kl;
  }
  const double ts = block_sum_t(ss, red), tk = block_sum_t(sk, red);
  if (threadIdx.x == 0) {
    a.part[((size_t)k * kLsBlocks + blockIdx.x) * 2 + 0] = ts;
    a.part[((size_t)k * kLsBlocks + blockIdx.x) * 2 + 1] = tk;
  }
}

// stable-baselines' sequential rule: the first k whose losses are finite, meankl <= 1.5 max_kl and optimgain - optimgain_before
// >= 0; none: theta_before stays.  Writes the losses after and SC_ACC.
__global__ void trpo_ls_select_kernel(const double* __restrict__ part, const float* __restrict__ lsc, int N, int A, float entcoeff,
                                      float max_kl, double* sc, float* met) {
  if (threadIdx.x != 0) return;
  if (sc[SC_ZERO] != 0.0 || sc[SC_BAD] != 0.0) { sc[SC_ACC] = sc[SC_ZERO] != 0.0 ? -2.0 : -1.0; return; }
  const float before = met[TM_BEFORE + 0];
  sc[SC_ACC] = -1.0;
  for (int k = 0; k < kNcand; ++k) {
    double su = 0.0, kl = 0.0;
    for (int b = 0; b < kLsBlocks; ++b) { su += part[((size_t)k * kLsBlocks + b) * 2]; kl += part[((size_t)k * kLsBlocks + b) * 2 + 1]; }
    su /= N; kl /= N;
    double ent = kHalfLog2PiE * A;
    for (int j = 0; j < A; ++j) ent += (double)lsc[(size_t)k * A + j];
    const float l[5] = {(float)(su + entcoeff * ent), (float)kl, (float)(entcoeff * ent), (float)su, (float)ent};
    bool fin = true;
    for (int q = 0; q < 5; ++q) fin = fin && isfinite(l[q]);
    if (!fin || l[1] > 1.5f * max_kl || l[0] - before < 0.f) continue;
    sc[SC_ACC] = k;
    for (int q = 0; q < 5; ++q) met[TM_AFTER + q] = l[q];
    break;
  }
}

// theta = theta_old + 0.5^k fullstep for the accepted k (the same rounding as the candidates)
__global__ void trpo_apply_kernel(float* __restrict__ P, const float* __restrict__ fs, int n, const double* __restrict__ sc) {
  const double acc = sc[SC_ACC];
  if (acc < 0.0) return;
  const float s = ldexpf(1.f, -(int)acc);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float f = fs[i];
    if (f != 0.f) P[i] = cand_value(P[i], f, s);
  }
}

struct VfTailArgs {
  const float* Y1;                   // [kVfBatch, H1] compact vf latent
  const float *Wvf, *bvf;
  const int* perm;                   // minibatch rows
  const float* ret;
  int H1;
  float* dZ1;                        // [kVfBatch, H1]
  float *gWvf, *gbvf;
  float* met;
  long long* counters;
  const double* sc;
};

// the value head of one minibatch: loss mean (V - R)^2, dV = 2 (V - R) / 128, the head's gradients and dZ1; advances the
// Adam step unless the iteration's step direction was not finite (trpo_vadam_kernel then applies nothing)
__global__ void __launch_bounds__(256) trpo_vf_tail_kernel(VfTailArgs a) {
  __shared__ float dv[kVfBatch];
  __shared__ double red[8];
  const int tid = threadIdx.x, H1 = a.H1;
  double l = 0.0;
  for (int r = tid; r < kVfBatch; r += blockDim.x) {
    float v = a.bvf[0];
    for (int k = 0; k < H1; ++k) v = fmaf(a.Y1[(size_t)r * H1 + k], a.Wvf[k], v);
    const float e = v - a.ret[a.perm[r]];
    l += (double)e * e;
    dv[r] = 2.f * e / (float)kVfBatch;
  }
  const double lt = block_sum_t(l, red);
  for (int i = tid; i < kVfBatch * H1; i += blockDim.x) {
    const int r = i / H1, k = i - r * H1;
    const float y = a.Y1[i];
    a.dZ1[i] = dv[r] * a.Wvf[k] * (1.f - y * y);
  }
  for (int k = tid; k <= H1; k += blockDim.x) {
    double g = 0.0;
    if (k < H1) {
      for (int r = 0; r < kVfBatch; ++r) g += (double)a.Y1[(size_t)r * H1 + k] * dv[r];
      a.gWvf[k] = (float)g;
    } else {
      for (int r = 0; r < kVfBatch; ++r) g += dv[r];
      a.gbvf[0] = (float)g;
    }
  }
  if (tid == 0) {
    a.met[TM_VF] += (float)(lt / kVfBatch);
    if (a.sc[SC_BAD] == 0.0) a.counters[0] += 1;
  }
}

struct VAdamArgs {
  float *P, *Mo, *Vo;
  const float* G;
  int64_t oW0, nW0, ob0, ob1, oW1, oWvf, obvf;   // ranges of the vf variables
  int H0, H1;
  int n;
  const long long* counters;
  const double* sc;
  float lr;
};

__device__ __forceinline__ bool vf_entry(const VAdamArgs& a, int64_t i) {
  if (i >= a.oW0 && i < a.oW0 + a.nW0) return (i - a.oW0) % (2 * a.H0) >= a.H0;   // W0's vf columns
  if (i >= a.ob0 && i < a.ob0 + 2 * a.H0) return i - a.ob0 >= a.H0;
  if (i >= a.oW1 && i < a.oW1 + (int64_t)a.H0 * a.H1) return true;
  if (i >= a.ob1 && i < a.ob1 + a.H1) return true;
  if (i >= a.oWvf && i < a.oWvf + a.H1) return true;
  return i == a.obvf;
}

// MpiAdam on the value variables: step = lr sqrt(1 - b2^t) / (1 - b1^t) m / (sqrt(v) + 1e-8); nothing after a failed CG check
__global__ void __launch_bounds__(256) trpo_vadam_kernel(VAdamArgs a) {
  if (a.sc[SC_BAD] != 0.0) return;
  const double t = (double)a.counters[0];
  const float lr = (float)((double)a.lr * sqrt(1.0 - pow(0.999, t)) / (1.0 - pow(0.9, t)));
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
    if (!vf_entry(a, i)) continue;
    const float g = a.G[i];
    const float m = 0.9f * a.Mo[i] + 0.1f * g;
    const float v = 0.999f * a.Vo[i] + 0.001f * (g * g);
    a.Mo[i] = m; a.Vo[i] = v;
    a.P[i] = a.P[i] - lr * m / (sqrtf(v) + kAdamEps);
  }
}

}  // namespace

// the backward launches of one tower over M rows: dZ1 (compact) -> weight / bias gradients of layer 1, dZ0 (compact), layer 0
struct TowerBwd { GemmGroup b1, b0; };
// the vf tower's forward over one value minibatch
struct VfFwd { GemmGroup l0, l1; };
struct VfMb { VfFwd f; TowerBwd b; const int* perm = nullptr; };
// the tangent launches of the Fisher-vector product
struct FvpLaunch { GemmGroup t0, t1; TowerBwd b; };

// network, rollout of E = 1 env, actor, update graph, counters [0] value-Adam step, [1] stream-1 step (actor_critic.cuh); Mo / Vo
// are the value Adam's moments, G the policy gradient g; h_buf holds metrics and scalars
struct b2g_trpo : ActorCritic {
  b2g_trpo_cfg cfg{};
  int N = 0, NF = 0, RMAX = 0, NVMB = 0;
  float* Gv = nullptr;              // value gradient
  float *X = nullptr, *Rv = nullptr, *Pv = nullptr, *Zv = nullptr, *FS = nullptr;   // CG vectors and the full step
  float *atarg = nullptr, *mu_old = nullptr, *nlp_old = nullptr, *sdm = nullptr, *sdls = nullptr, *u = nullptr;
  float *dZ1 = nullptr, *dZ0 = nullptr, *T0 = nullptr, *T1 = nullptr;
  float *dZls = nullptr, *Y0c = nullptr, *Y1c = nullptr, *cand = nullptr;
  float *vZ0 = nullptr, *vY0 = nullptr, *vY1 = nullptr, *vdZ1 = nullptr, *vdZ0 = nullptr;
  int *perm = nullptr, *vrowoff = nullptr;
  double *part = nullptr, *amax = nullptr, *lspart = nullptr, *sc = nullptr;
  float* met = nullptr;
  AcFwd f_all;
  TowerBwd gbwd;
  FvpLaunch fvp;
  GemmGroup ls_dz, ls_l1;
  std::vector<VfMb> vmbs;
  bool carried = false;             // rollout row 0 holds the boundary observation and action of the last update
};

namespace {

using Tab = AcTab;
static_assert(TM_N + 2 * SC_N <= kAcHostFloats, "h_buf holds the metrics and the scalars");
// the policy variables pi_fc0, pi_fc1 and pi (zip entries 0, 1, 4, 5, 10, 11, 12): the gradient arena of the policy step
constexpr uint32_t kGradMask = (1u << 0) | (1u << 1) | (1u << 4) | (1u << 5) | (1u << 10) | (1u << 11) | (1u << 12);

// tower tw's backward over M rows: obs rows xrows, layer-0 outputs at y0 (rows y0rows, tower column base applied), compact dZ1 /
// dZ0; gradients into the arena `out`
int make_tower_bwd(b2g_trpo* h, TowerBwd& bw, int tw, int M, const float* obs, const int* xrows, const float* y0, const int* y0rows,
                   float* dZ1, float* dZ0, float* out, Tab& tab) {
  const int D = h->D, H0 = h->H0, H1 = h->H1;
  bw.b1 = GemmGroup(); bw.b0 = GemmGroup();
  bw.b1.name = "trpo_l1_bwd"; bw.b0.name = "trpo_l0_wgrad";
  const int tiles1 = ((H0 + 63) / 64) * ((H1 + 63) / 64);
  GemmDesc w = gemm_desc(y0, tab["iH0"], y0rows, dZ1, tab["rM_H1"], tab["iH1"], out + h->oW1[tw], tab["iH0_H1"], tab["iH1"], H0, H1, M,
                         GG_COLSUM | GG_EPI_ATOMIC, ac_splits_for(tiles1, M));
  w.colsum = out + h->ob1[tw];
  bw.b1.host.push_back(w);
  GemmDesc dg = gemm_desc(dZ1, tab["rM_H1"], tab["iH1"], h->P + h->oW1[tw], tab["iH1"], tab["iH0_H1"], dZ0, tab["rM_H0"], tab["iH0"], M, H0,
                          H1, GG_A_RVEC | GG_B_RVEC | GG_EPI_TANH_GRAD);
  dg.mask = y0; dg.kM = y0rows; dg.kN = tab["iH0"];
  bw.b1.host.push_back(dg);
  const int tiles0 = ((D + 63) / 64) * ((H0 + 63) / 64);
  GemmDesc w0 = gemm_desc(obs, tab["iD"], xrows, dZ0, tab["rM_H0"], tab["iH0"], out + h->oW0 + tw * H0, tab["iD_2H0"], tab["iH0"], D, H0, M,
                          GG_COLSUM | GG_EPI_ATOMIC, ac_splits_for(tiles0, M));
  w0.colsum = out + h->ob0 + tw * H0;
  bw.b0.host.push_back(w0);
  if (int rc = finalize_tiles(bw.b1, h->allocs, h->stream)) return rc;
  return finalize_tiles(bw.b0, h->allocs, h->stream);
}

void tower_bwd_issue(const TowerBwd& bw, cudaStream_t s) {
  gg_simt_launch_tanh(bw.b1.dev, (int)bw.b1.host.size(), bw.b1.total_tiles, s);
  gg_simt_launch(bw.b0.dev, (int)bw.b0.host.size(), bw.b0.total_tiles, s);
}

int make_vf_mb(b2g_trpo* h, VfMb& mb, const int* xrows, const int* perm, Tab& tab) {
  const int D = h->D, H0 = h->H0, H1 = h->H1, M = kVfBatch;
  mb.perm = perm;
  mb.f.l0 = GemmGroup(); mb.f.l1 = GemmGroup();
  mb.f.l0.name = "trpo_vf_l0"; mb.f.l1.name = "trpo_vf_l1";
  const int tiles = ((M + 63) / 64) * ((H0 + 63) / 64);
  mb.f.l0.host.push_back(gemm_desc(h->r_obs, xrows, tab["iD"], h->P + h->oW0 + H0, tab["iD_2H0"], tab["iH0"], h->vZ0, tab["rM_H0"], tab["iH0"],
                                   M, H0, D, GG_A_RVEC | GG_EPI_ATOMIC, ac_splits_for(tiles, D)));
  GemmDesc g = gemm_desc(h->vY0, tab["rM_H0"], tab["iH0"], h->P + h->oW1[1], tab["iH0_H1"], tab["iH1"], h->vY1, tab["rM_H1"], tab["iH1"], M, H1,
                         H0, GG_A_RVEC | GG_EPI_BIAS_TANH);
  g.bias = h->P + h->ob1[1];
  mb.f.l1.host.push_back(g);
  if (int rc = finalize_tiles(mb.f.l0, h->allocs, h->stream)) return rc;
  if (int rc = finalize_tiles(mb.f.l1, h->allocs, h->stream)) return rc;
  return make_tower_bwd(h, mb.b, 1, M, h->r_obs, xrows, h->vY0, tab["rM_H0"], h->vdZ1, h->vdZ0, h->Gv, tab);
}

int make_fvp(b2g_trpo* h, Tab& tab) {
  const int D = h->D, H0 = h->H0, H1 = h->H1, M = h->NF;
  FvpLaunch& f = h->fvp;
  f.t0 = GemmGroup(); f.t1 = GemmGroup();
  f.t0.name = "trpo_fvp_t0"; f.t1.name = "trpo_fvp_t1";
  const int tiles = ((M + 63) / 64) * ((H0 + 63) / 64);
  f.t0.host.push_back(gemm_desc(h->r_obs, tab["x5"], tab["iD"], h->Pv + h->oW0, tab["iD_2H0"], tab["iH0"], h->T0, tab["rM_H0"], tab["iH0"], M,
                                H0, D, GG_A_RVEC | GG_EPI_ATOMIC, ac_splits_for(tiles, D)));
  f.t1.host.push_back(gemm_desc(h->T0, tab["rM_H0"], tab["iH0"], h->P + h->oW1[0], tab["iH0_H1"], tab["iH1"], h->T1, tab["rM_H1"], tab["iH1"],
                                M, H1, H0, GG_A_RVEC | GG_EPI_ATOMIC));
  f.t1.host.push_back(gemm_desc(h->Y0, tab["y0_5"], tab["iH0"], h->Pv + h->oW1[0], tab["iH0_H1"], tab["iH1"], h->T1, tab["rM_H1"], tab["iH1"],
                                M, H1, H0, GG_A_RVEC | GG_EPI_ATOMIC));
  if (int rc = finalize_tiles(f.t0, h->allocs, h->stream)) return rc;
  if (int rc = finalize_tiles(f.t1, h->allocs, h->stream)) return rc;
  return make_tower_bwd(h, f.b, 0, M, h->r_obs, tab["x5"], h->Y0, tab["y0_5"], h->dZ1, h->dZ0, h->Zv, tab);
}

int make_ls(b2g_trpo* h, Tab& tab) {
  const int D = h->D, H0 = h->H0, H1 = h->H1, N = h->N;
  h->ls_dz = GemmGroup(); h->ls_l1 = GemmGroup();
  h->ls_dz.name = "trpo_ls_dz"; h->ls_l1.name = "trpo_ls_l1";
  const int tiles = ((N + 63) / 64) * ((H0 + 63) / 64);
  h->ls_dz.host.push_back(gemm_desc(h->r_obs, tab["xall"], tab["iD"], h->FS + h->oW0, tab["iD_2H0"], tab["iH0"], h->dZls, tab["rM_H0"],
                                    tab["iH0"], N, H0, D, GG_A_RVEC | GG_EPI_ATOMIC, ac_splits_for(tiles, D)));
  float* W1c = h->cand + (size_t)kNcand * H0;
  float* b1c = W1c + (size_t)kNcand * H0 * H1;
  for (int k = 0; k < kNcand; ++k) {
    GemmDesc g = gemm_desc(h->Y0c + (size_t)k * N * H0, tab["rM_H0"], tab["iH0"], W1c + (size_t)k * H0 * H1, tab["iH0_H1"], tab["iH1"],
                           h->Y1c + (size_t)k * N * H1, tab["rM_H1"], tab["iH1"], N, H1, H0, GG_A_RVEC | GG_EPI_BIAS_TANH);
    g.bias = b1c + (size_t)k * H1;
    h->ls_l1.host.push_back(g);
  }
  if (int rc = finalize_tiles(h->ls_dz, h->allocs, h->stream)) return rc;
  return finalize_tiles(h->ls_l1, h->allocs, h->stream);
}

int grid_for(int64_t n, int threads = 256) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + threads - 1) / threads, 1 << 20)); }

void dot_issue(b2g_trpo* h, const float* a, const float* b, bool with_max, cudaStream_t s) {
  trpo_dot_kernel<<<kDotBlocks, kDotThreads, 0, s>>>(a, b, (int)h->n_train, h->part, with_max ? h->amax : nullptr);
}

void cg_stage(b2g_trpo* h, int stage, cudaStream_t s) { trpo_conjgrad_kernel<<<1, 32, 0, s>>>(stage, h->part, h->amax, h->sc, h->met, h->cfg.max_kl); }

void vec_issue(b2g_trpo* h, int op, cudaStream_t s) {
  trpo_vec_kernel<<<grid_for(h->n_train), 256, 0, s>>>(op, (int)h->n_train, h->sc, h->G, h->X, h->Rv, h->Pv, h->Zv, h->FS);
}

// Zv = F Pv over the rows [::5] (the forward at theta_old over the batch is in Z0 / Y0 / Y1)
void fvp_issue(b2g_trpo* h, cudaStream_t s) {
  const int M = h->NF, H0 = h->H0, H1 = h->H1, A = h->A;
  const FvpLaunch& f = h->fvp;
  cudaMemsetAsync(h->T0, 0, (size_t)M * H0 * sizeof(float), s);
  cudaMemsetAsync(h->T1, 0, (size_t)M * H1 * sizeof(float), s);
  cudaMemsetAsync(h->Zv, 0, (size_t)h->n_train * sizeof(float), s);
  gg_simt_launch(f.t0.dev, (int)f.t0.host.size(), f.t0.total_tiles, s);
  trpo_tangent_kernel<<<grid_for((int64_t)M * H0), 256, 0, s>>>(h->T0, h->Pv + h->ob0, h->Y0, 5 * 2 * H0, M, H0);
  gg_simt_launch(f.t1.dev, (int)f.t1.host.size(), f.t1.total_tiles, s);
  trpo_tangent_kernel<<<grid_for((int64_t)M * H1), 256, 0, s>>>(h->T1, h->Pv + h->ob1[0], h->Y1, 5 * 2 * H1, M, H1);
  trpo_fvp_head_kernel<<<grid_for(M, 128), 128, 0, s>>>(h->T1, h->Y1, 5 * 2 * H1, h->P + h->oWpi, h->Pv + h->oWpi, h->Pv + h->obpi,
                                                        h->P + h->ols, M, H1, A, h->u);
  trpo_head_bwd_kernel<<<grid_for((int64_t)M * H1), 256, 0, s>>>(h->u, h->P + h->oWpi, h->Y1, 5 * 2 * H1, M, H1, A, h->dZ1);
  tower_bwd_issue(f.b, s);
  trpo_headgrad_kernel<<<H1 * A + A, 256, 0, s>>>(h->Y1, 5 * 2 * H1, h->u, nullptr, 0.f, M, H1, A, h->Zv + h->oWpi, h->Zv + h->obpi, nullptr);
  trpo_fvp_finish_kernel<<<grid_for(h->n_train), 256, 0, s>>>(h->Zv, h->Pv, (int)h->n_train, h->ols, A, h->cfg.cg_damping);
}

// oldpi := pi, the policy gradient g at theta_old over rollout rows 0..N-1, and CG's start: x = 0, r = p = g
void policy_grad_issue(b2g_trpo* h, cudaStream_t s) {
  const int N = h->N, H1 = h->H1, A = h->A;
  const b2g_trpo_cfg& c = h->cfg;
  // oldpi := pi
  cudaMemcpyAsync(h->P + h->n_total, h->P, (size_t)h->n_total * sizeof(float), cudaMemcpyDeviceToDevice, s);
  cudaMemsetAsync(h->met, 0, TM_N * sizeof(float), s);
  // ---- the gradient at theta_old
  ac_fwd_issue(h, h->f_all, s);
  PrepArgs pa{};
  pa.h = ac_head_args(h); pa.N = N; pa.act = h->r_act; pa.adv = h->r_adv; pa.entcoeff = c.entcoeff;
  pa.atarg = h->atarg; pa.mu_old = h->mu_old; pa.nlp_old = h->nlp_old; pa.sdm = h->sdm; pa.sdls = h->sdls; pa.met = h->met;
  trpo_prep_kernel<<<1, kPrepThreads, 0, s>>>(pa);
  cudaMemsetAsync(h->G, 0, (size_t)h->n_train * sizeof(float), s);
  trpo_head_bwd_kernel<<<grid_for((int64_t)N * H1), 256, 0, s>>>(h->sdm, h->P + h->oWpi, h->Y1, 2 * H1, N, H1, A, h->dZ1);
  tower_bwd_issue(h->gbwd, s);
  trpo_headgrad_kernel<<<H1 * A + 2 * A, 256, 0, s>>>(h->Y1, 2 * H1, h->sdm, h->sdls, c.entcoeff, N, H1, A, h->G + h->oWpi, h->G + h->obpi,
                                                      h->G + h->ols);
  // ---- conjugate gradient on F x = g
  dot_issue(h, h->G, h->G, true, s);
  cg_stage(h, CG_INIT, s);
  vec_issue(h, 0, s);
}

// one CG iteration: z = F p, alpha, x += alpha p, r -= alpha z, beta, p = r + beta p
void cg_iteration_issue(b2g_trpo* h, cudaStream_t s) {
  fvp_issue(h, s);
  dot_issue(h, h->Pv, h->Zv, false, s);
  cg_stage(h, CG_ALPHA, s);
  vec_issue(h, 1, s);
  dot_issue(h, h->Rv, h->Rv, false, s);
  cg_stage(h, CG_BETA, s);
  vec_issue(h, 2, s);
}

// the policy and value step on rollout rows 0..N-1 (obs, actions, raw advantages r_adv, tdlamret r_ret) and the uploaded
// permutation
void core_issue(b2g_trpo* h, cudaStream_t s) {
  const int N = h->N, H0 = h->H0, H1 = h->H1, A = h->A;
  const b2g_trpo_cfg& c = h->cfg;
  policy_grad_issue(h, s);
  for (int it = 0; it < c.cg_iters; ++it) cg_iteration_issue(h, s);
  dot_issue(h, h->X, h->X, false, s);
  cg_stage(h, CG_CHECK, s);
  cudaMemcpyAsync(h->Pv, h->X, (size_t)h->n_train * sizeof(float), cudaMemcpyDeviceToDevice, s);
  fvp_issue(h, s);
  dot_issue(h, h->X, h->Zv, false, s);
  cg_stage(h, CG_SHS, s);
  vec_issue(h, 3, s);
  dot_issue(h, h->G, h->FS, false, s);
  cg_stage(h, CG_EI, s);
  // ---- line search: ten candidates in one pass
  CandArgs ca{};
  ca.P = h->P; ca.fs = h->FS; ca.ob0 = h->ob0; ca.oW1 = h->oW1[0]; ca.ob1 = h->ob1[0]; ca.oWpi = h->oWpi; ca.obpi = h->obpi; ca.ols = h->ols;
  ca.H0 = H0; ca.H1 = H1; ca.A = A;
  ca.b0c = h->cand; ca.W1c = ca.b0c + (size_t)kNcand * H0; ca.b1c = ca.W1c + (size_t)kNcand * H0 * H1;
  ca.Wpic = ca.b1c + (size_t)kNcand * H1; ca.bpic = ca.Wpic + (size_t)kNcand * H1 * A; ca.lsc = ca.bpic + (size_t)kNcand * A;
  trpo_cand_kernel<<<dim3(grid_for(H0 + H0 * H1 + H1 + H1 * A + 2 * A), kNcand), 256, 0, s>>>(ca);
  cudaMemsetAsync(h->dZls, 0, (size_t)N * H0 * sizeof(float), s);
  gg_simt_launch(h->ls_dz.dev, (int)h->ls_dz.host.size(), h->ls_dz.total_tiles, s);
  trpo_ls_l0_kernel<<<dim3(std::min(grid_for((int64_t)N * H0), 1024), kNcand), 256, 0, s>>>(h->Z0, 2 * H0, h->dZls, ca.b0c, N, H0, h->Y0c);
  gg_simt_launch_tanh(h->ls_l1.dev, (int)h->ls_l1.host.size(), h->ls_l1.total_tiles, s);
  LsArgs la{};
  la.Y1c = h->Y1c; la.Wpic = ca.Wpic; la.bpic = ca.bpic; la.lsc = ca.lsc;
  la.mu_old = h->mu_old; la.nlp_old = h->nlp_old; la.atarg = h->atarg; la.act = h->r_act; la.ls_old = h->P + h->ols;
  la.N = N; la.H1 = H1; la.A = A; la.part = h->lspart;
  trpo_ls_loss_kernel<<<dim3(kLsBlocks, kNcand), kLsThreads, 0, s>>>(la);
  trpo_ls_select_kernel<<<1, 32, 0, s>>>(h->lspart, ca.lsc, N, A, c.entcoeff, c.max_kl, h->sc, h->met);
  trpo_apply_kernel<<<grid_for(h->n_train), 256, 0, s>>>(h->P, h->FS, (int)h->n_train, h->sc);
  // ---- value step
  const int nperm = c.vf_iters * N;
  if (nperm > 0) trpo_rows_kernel<<<grid_for(nperm), 256, 0, s>>>(h->perm, nperm, h->XS, h->vrowoff);
  VAdamArgs va{};
  va.P = h->P; va.Mo = h->Mo; va.Vo = h->Vo; va.G = h->Gv;
  va.oW0 = h->oW0; va.nW0 = (int64_t)h->D * 2 * H0; va.ob0 = h->ob0; va.ob1 = h->ob1[1]; va.oW1 = h->oW1[1]; va.oWvf = h->oWvf; va.obvf = h->obvf;
  va.H0 = H0; va.H1 = H1; va.n = (int)h->n_train; va.counters = h->counters; va.sc = h->sc; va.lr = c.vf_stepsize;
  for (const VfMb& mb : h->vmbs) {
    cudaMemsetAsync(h->Gv, 0, (size_t)h->n_train * sizeof(float), s);
    cudaMemsetAsync(h->vZ0, 0, (size_t)kVfBatch * H0 * sizeof(float), s);
    gg_simt_launch(mb.f.l0.dev, (int)mb.f.l0.host.size(), mb.f.l0.total_tiles, s);
    ac_bias_tanh(h->vZ0, h->P + h->ob0 + H0, h->vY0, kVfBatch, H0, s);
    gg_simt_launch_tanh(mb.f.l1.dev, (int)mb.f.l1.host.size(), mb.f.l1.total_tiles, s);
    VfTailArgs ta{};
    ta.Y1 = h->vY1; ta.Wvf = h->P + h->oWvf; ta.bvf = h->P + h->obvf; ta.perm = mb.perm; ta.ret = h->r_ret; ta.H1 = H1; ta.dZ1 = h->vdZ1;
    ta.gWvf = h->Gv + h->oWvf; ta.gbvf = h->Gv + h->obvf; ta.met = h->met; ta.counters = h->counters; ta.sc = h->sc;
    trpo_vf_tail_kernel<<<1, 256, 0, s>>>(ta);
    tower_bwd_issue(mb.b, s);
    trpo_vadam_kernel<<<std::max(1, std::min(264, grid_for(h->n_train))), 256, 0, s>>>(va);
  }
}

// the whole iteration after the uploads: boundary action and bootstrap value, GAE, the step, then row 0 of the next batch
int update_issue(b2g_trpo* h) {
  cudaStream_t s = h->stream;
  const int N = h->N, A = h->A;
  ac_fwd_issue(h, h->f_boot, s);
  AcActArgs a = ac_act_args(h, 1, 0);
  a.t = N;
  ac_act(a, s);
  ac_gae(h->r_rew, h->r_val, h->r_done, h->r_val + N, N, 1, h->cfg.gamma, h->cfg.lam, h->r_adv, h->r_ret, s);
  core_issue(h, s);
  ac_fwd_issue(h, h->f_boot, s);
  AcActArgs v = ac_act_args(h, 1, 1);
  v.lastv = h->r_val;                 // row 0's value under the updated value tower
  ac_act(v, s);
  cudaMemcpyAsync(h->r_obs, h->r_obs + (size_t)N * h->XS, (size_t)h->XS * sizeof(float), cudaMemcpyDeviceToDevice, s);
  cudaMemcpyAsync(h->r_act, h->r_act + (size_t)N * A, (size_t)A * sizeof(float), cudaMemcpyDeviceToDevice, s);
  cudaMemcpyAsync(h->r_nlp, h->r_nlp + N, sizeof(float), cudaMemcpyDeviceToDevice, s);
  cudaMemcpyAsync(h->r_done, h->r_done + N, sizeof(float), cudaMemcpyDeviceToDevice, s);
  CK(cudaGetLastError());
  return 0;
}

// metrics; B2G_ESTATE when the step direction was not finite
int fetch(b2g_trpo* h, b2g_trpo_metrics* out) {
  CK(cudaMemcpyAsync(h->h_buf, h->met, TM_N * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  double* hs = reinterpret_cast<double*>(h->h_buf + TM_N);
  CK(cudaMemcpyAsync(hs, h->sc, SC_N * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  const float* m = h->h_buf;
  if (out) {
    out->optimgain = m[0]; out->meankl = m[1]; out->entbonus = m[2]; out->surrgain = m[3]; out->entropy = m[4];
    out->optimgain_after = m[5]; out->meankl_after = m[6]; out->entbonus_after = m[7]; out->surrgain_after = m[8]; out->entropy_after = m[9];
    out->grad_sq = m[TM_GG]; out->shs = m[TM_SHS]; out->expected_improve = m[TM_EI];
    out->vf_loss = h->vmbs.empty() ? 0.f : m[TM_VF] / (float)h->vmbs.size();
    out->cg_iters = (int32_t)hs[SC_ITERS]; out->accepted = (int32_t)hs[SC_ACC];
    out->n_iterations = h->n_updates;
  }
  if (hs[SC_BAD] != 0.0) return b2g_fail(B2G_ESTATE, "the conjugate-gradient step direction is not finite");
  return 0;
}

// the policy variables (var_list order: the gradient arena's entries in zip order) <-> the arena layout of the gradient / CG
// vectors
void flat_arena(const b2g_trpo* h, float* flat, float* arena, bool to_arena) {
  size_t k = 0;
  for (const ParamEntry& e : h->params.entries()) {
    if (!e.grad) continue;
    for (int64_t r = 0; r < e.rows; ++r)
      for (int64_t c = 0; c < e.cols; ++c, ++k) {
        float& a = arena[e.off + r * e.stride + c];
        if (to_arena) a = flat[k]; else flat[k] = a;
      }
  }
}

int download_flat(b2g_trpo* h, const float* dev, float* flat) {
  std::vector<float> host((size_t)h->n_train);
  CK(cudaMemcpyAsync(host.data(), dev, host.size() * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  flat_arena(h, flat, host.data(), false);
  return 0;
}

}  // namespace

extern "C" {

int b2g_trpo_destroy(b2g_trpo* h) {
  if (!h) return 0;
  ac_release(h);
  delete h;
  return 0;
}

int b2g_trpo_create(const b2g_trpo_cfg* cfg, b2g_trpo** out) {
  if (!cfg || !out) return b2g_fail(B2G_EINVAL, "cfg/out is NULL");
  *out = nullptr;
  const b2g_trpo_cfg& c = *cfg;
  if (int rc = ac_check_net(c.obs_dim, c.n_actions, c.hidden0, c.hidden1)) return rc;
  if (c.timesteps_per_batch < 1 || c.timesteps_per_batch > kMaxN) return b2g_fail(B2G_EINVAL, "timesteps_per_batch must be in [1, 16384]");
  if (c.cg_iters < 1 || c.cg_iters > 64) return b2g_fail(B2G_EINVAL, "cg_iters must be in [1, 64]");
  if (c.vf_iters < 0 || c.vf_iters > 64) return b2g_fail(B2G_EINVAL, "vf_iters must be in [0, 64]");
  if (!(c.max_kl > 0.f)) return b2g_fail(B2G_EINVAL, "max_kl must be > 0");
  if (!(c.cg_damping >= 0.f) || !(c.vf_stepsize >= 0.f)) return b2g_fail(B2G_EINVAL, "cg_damping and vf_stepsize must be >= 0");
  const int64_t XS = ac_row_stride(c.obs_dim);
  if ((int64_t)(c.timesteps_per_batch + 1) * XS >= (1LL << 31))
    return b2g_fail(B2G_EINVAL, "rollout (timesteps_per_batch + 1) * obs_dim must be < 2^31 floats");
  if (int rc = check_device(c.device)) return rc;
  const int64_t N = c.timesteps_per_batch, H0 = c.hidden0, H1 = c.hidden1;
  {   // the line search's candidate activations: kNcand * N * (H0 + H1) floats
    const size_t ls_bytes = (size_t)kNcand * N * (H0 + H1) * sizeof(float);
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) return b2g_fail(B2G_ECUDA, "cudaMemGetInfo");
    if (ls_bytes + ((size_t)N + 1) * XS * sizeof(float) > free_b)
      return b2g_fail(B2G_EINVAL, "the rollout and the line-search scratch (" + std::to_string(ls_bytes >> 20) + " MB) do not fit the " +
                                      std::to_string(free_b >> 20) + " MB of free device memory");
  }
  b2g_trpo* h = new b2g_trpo();
  h->cfg = c;
  auto bail = [&](int rc) { std::string keep = g_b2g_err; b2g_trpo_destroy(h); g_b2g_err = keep; return rc; };
  if (int rc = ac_init(h, c.device, c.obs_dim, c.n_actions, c.hidden0, c.hidden1, 1, (int)N, 64, c.seed)) return bail(rc);
  h->rms.set_call = "b2g_trpo_obs_rms_set";
  h->N = (int)N; h->NF = (int)((N + 4) / 5);
  h->RMAX = (int)std::max<int64_t>(N + 1, h->P_ROWS);
  h->NVMB = c.vf_iters * (int)(N / kVfBatch);
  const int A = h->A;
  // zip order: pi/model/... (PPO2's creation order), then the same under oldpi/model/ (a second copy of the whole block)
  ac_layout(h, "pi/model/", kGradMask, 2);
  h->params.add_copies(0, 15, "pi/model/", "oldpi/model/", h->n_total);
  Tab tab;
  int rc = ac_alloc(h, h->RMAX, tab);
  if (rc) return bail(rc);
  const int64_t R = h->RMAX, NF = h->NF;
#define DA(ptr, count) if ((rc = dev_alloc(h->allocs, h->stream, &(ptr), (size_t)(count)))) return bail(rc)
  DA(h->Gv, h->n_train);
  DA(h->X, h->n_train); DA(h->Rv, h->n_train); DA(h->Pv, h->n_train); DA(h->Zv, h->n_train); DA(h->FS, h->n_train);
  DA(h->atarg, N); DA(h->mu_old, N * A); DA(h->nlp_old, N); DA(h->sdm, N * A); DA(h->sdls, N * A); DA(h->u, NF * A);
  DA(h->dZ1, R * H1); DA(h->dZ0, R * H0); DA(h->T0, NF * H0); DA(h->T1, NF * H1);
  DA(h->dZls, N * H0); DA(h->Y0c, kNcand * N * H0); DA(h->Y1c, kNcand * N * H1);
  DA(h->cand, (int64_t)kNcand * (H0 + H0 * H1 + H1 + H1 * A + 2 * A));
  DA(h->vZ0, kVfBatch * H0); DA(h->vY0, kVfBatch * H0); DA(h->vY1, kVfBatch * H1); DA(h->vdZ1, kVfBatch * H1); DA(h->vdZ0, kVfBatch * H0);
  const int64_t nperm = std::max<int64_t>(1, (int64_t)c.vf_iters * N);
  DA(h->perm, nperm); DA(h->vrowoff, nperm);
  DA(h->part, kDotBlocks); DA(h->amax, kDotBlocks); DA(h->lspart, kNcand * kLsBlocks * 2); DA(h->sc, SC_N);
  DA(h->met, TM_N);
#undef DA
  auto T_ = [&](const char* nm, const std::vector<int>& v) {
    const int* p = nullptr;
    if (int r2 = upload_table(h->allocs, h->stream, v, &p)) return r2;
    tab[nm] = p;
    return 0;
  };
  if ((rc = T_("rM_H0", iota_tab((int)R, (int)H0))) || (rc = T_("rM_H1", iota_tab((int)R, (int)H1))) ||
      (rc = T_("xall", iota_tab((int)N, h->XS))) || (rc = T_("x5", iota_tab((int)NF, 5 * h->XS))) ||
      (rc = T_("y0_5", iota_tab((int)NF, 5 * 2 * (int)H0))))
    return bail(rc);
  if ((rc = ac_make_fwd(h, h->f_all, h->r_obs, tab["xall"], (int)N, tab))) return bail(rc);
  if ((rc = make_tower_bwd(h, h->gbwd, 0, (int)N, h->r_obs, tab["xall"], h->Y0, tab["rM_2H0"], h->dZ1, h->dZ0, h->G, tab))) return bail(rc);
  if ((rc = make_fvp(h, tab))) return bail(rc);
  if ((rc = make_ls(h, tab))) return bail(rc);
  h->vmbs.resize(h->NVMB);
  const int per_pass = (int)(N / kVfBatch);
  for (int k = 0; k < h->NVMB; ++k) {
    const int64_t first = (int64_t)(k / per_pass) * N + (int64_t)(k % per_pass) * kVfBatch;   // contiguous, the partial batch dropped
    if ((rc = make_vf_mb(h, h->vmbs[k], h->vrowoff + first, h->perm + first, tab))) return bail(rc);
  }
  if (cudaStreamSynchronize(h->stream) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "create sync"));
  *out = h;
  return 0;
}

int b2g_trpo_param_count(const b2g_trpo* h) { return param_count(h); }
int b2g_trpo_param_info(const b2g_trpo* h, int idx, char* name, size_t name_cap, int64_t* rows, int64_t* cols, int32_t* ndim) {
  return param_info(h, idx, name, name_cap, rows, cols, ndim);
}
int b2g_trpo_get_param(b2g_trpo* h, const char* name, float* dst, size_t numel) { return param_copy(h, name, ParamCopy::Get, dst, numel); }
int b2g_trpo_set_param(b2g_trpo* h, const char* name, const float* src, size_t numel) {
  return param_copy(h, name, ParamCopy::Set, const_cast<float*>(src), numel);
}
int b2g_trpo_get_grad(b2g_trpo* h, const char* name, float* dst, size_t numel) { return param_copy(h, name, ParamCopy::GetGrad, dst, numel); }

int b2g_trpo_rollout_act(b2g_trpo* h, const float* obs, float* act_out) {
  B2G_USABLE(h);
  if (!h || !obs || !act_out) return b2g_fail(B2G_EINVAL, "NULL argument");
  if (h->t >= h->N) return b2g_fail(B2G_ESTATE, "the rollout holds timesteps_per_batch rows: call b2g_trpo_update first");
  if (h->t > 0 || !h->carried) return ac_rollout_act(h, obs, act_out);
  // row 0 after an update: the boundary action drawn before it
  CK(cudaSetDevice(h->device));
  if (int rc = ac_upload_rows(h, h->r_obs, obs, 1)) return rc;
  CK(cudaMemcpyAsync(act_out, h->r_act, (size_t)h->A * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->acted = true;
  h->ob_n = 0;
  return 0;
}

int b2g_trpo_rollout_reward(b2g_trpo* h, float rew, float done) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  if (h->t >= h->N) return b2g_fail(B2G_ESTATE, "the rollout holds timesteps_per_batch rows: call b2g_trpo_update first");
  return ac_rollout_reward(h, &rew, &done);
}

int b2g_trpo_rollout_reset(b2g_trpo* h) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  if (int rc = ac_rollout_reset(h)) return rc;
  h->carried = false;
  return 0;
}

int b2g_trpo_rollout_get(b2g_trpo* h, float* adv, float* ret, float* val, float* act) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  return ac_rollout_get(h, adv, ret, val, nullptr, act);
}

static int upload_perm(b2g_trpo* h, const int32_t* perm) {
  const int64_t n = (int64_t)h->cfg.vf_iters * h->N;
  for (int64_t i = 0; i < n; ++i)
    if (perm[i] < 0 || perm[i] >= h->N) return b2g_fail(B2G_EINVAL, "permutation entry " + std::to_string(i) + " is outside [0, N)");
  if (n > 0) CK(cudaMemcpyAsync(h->perm, perm, n * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
  return 0;
}

int b2g_trpo_update(b2g_trpo* h, const float* last_obs, const int32_t* perm, b2g_trpo_metrics* out) {
  B2G_USABLE(h);
  if (!h || (!perm && h->cfg.vf_iters > 0)) return b2g_fail(B2G_EINVAL, "NULL argument");
  if (h->t != h->N) return b2g_fail(B2G_ESTATE, "the rollout is not full: timesteps_per_batch rollout steps come before an update");
  if (int rc = ac_check_last_obs(h, last_obs)) return rc;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  if (int rc = upload_perm(h, perm)) return rc;
  if (int rc = ac_update_last_obs(h, last_obs)) return rc;
  if (int rc = ac_run_update(h, [&] { return update_issue(h); })) return rc;
  h->n_updates += 1;
  h->t = 0;
  h->carried = true;
  if (int rc = ac_update_finish(h, last_obs, false)) return rc;     // the update carried row N into row 0 itself
  return fetch(h, out);
}

int b2g_trpo_step_explicit(b2g_trpo* h, const float* obs, const float* actions, const float* adv, const float* tdlamret,
                           const int32_t* perm, b2g_trpo_metrics* out, float* grad, float* stepdir, float* fullstep) {
  B2G_USABLE(h);
  if (!h || !obs || !actions || !adv || !tdlamret || (!perm && h->cfg.vf_iters > 0)) return b2g_fail(B2G_EINVAL, "NULL argument");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  if (int rc = upload_perm(h, perm)) return rc;
  const size_t N = h->N;
  if (int rc = ac_upload_rows(h, h->r_obs, obs, h->N)) return rc;
  CK(cudaMemcpyAsync(h->r_act, actions, N * h->A * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaMemcpyAsync(h->r_adv, adv, N * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaMemcpyAsync(h->r_ret, tdlamret, N * sizeof(float), cudaMemcpyDefault, h->stream));
  core_issue(h, h->stream);
  CK(cudaGetLastError());
  h->n_updates += 1;
  h->t = 0;
  h->carried = false;
  h->acted = false;
  h->ob_n = 0;
  const int rc = fetch(h, out);
  if (grad) if (int r2 = download_flat(h, h->G, grad)) return r2;
  if (stepdir) if (int r2 = download_flat(h, h->X, stepdir)) return r2;
  if (fullstep) if (int r2 = download_flat(h, h->FS, fullstep)) return r2;
  return rc;
}

int b2g_trpo_fvp(b2g_trpo* h, const float* obs, const float* v, float* out) {
  B2G_USABLE(h);
  if (!h || !obs || !v || !out) return b2g_fail(B2G_EINVAL, "NULL argument");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  std::vector<float> arena((size_t)h->n_train, 0.f);
  flat_arena(h, const_cast<float*>(v), arena.data(), true);
  CK(cudaMemcpyAsync(h->Pv, arena.data(), arena.size() * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  if (int rc = ac_upload_rows(h, h->r_obs, obs, h->N)) return rc;
  ac_fwd_issue(h, h->f_all, h->stream);
  fvp_issue(h, h->stream);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(h->stream));
  h->t = 0;
  h->carried = false;
  h->acted = false;
  h->ob_n = 0;
  return download_flat(h, h->Zv, out);
}

int b2g_trpo_act(b2g_trpo* h, const float* obs, int n, int deterministic, float* act_out, float* value_out) {
  B2G_USABLE(h);
  if (!h || !obs || !act_out || n < 0) return b2g_fail(B2G_EINVAL, "bad argument");
  return ac_predict(h, obs, n, deterministic, act_out, value_out, nullptr);
}

int b2g_trpo_get_step(b2g_trpo* h, int64_t* adam_step, int64_t* noise_step, int32_t* rollout_rows) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  return ac_get_step(h, adam_step, noise_step, rollout_rows);
}

// ---- VecNormalize's obs_rms on the device and the observe path (bodies in actor_critic.cu); the boundary row carried into
// row 0 is the normalised row as it was staged
#define B2G_TRPO_HANDLE(h) B2G_USABLE(h); if (!h) return b2g_fail(B2G_EINVAL, "NULL handle")
int b2g_trpo_obs_rms_set(b2g_trpo* h, const double* mean, const double* var, double count) { return ac_obs_rms_set(h, mean, var, count); }
int b2g_trpo_obs_rms_get(b2g_trpo* h, double* mean, double* var, double* count) { return ac_obs_rms_get(h, mean, var, count); }
int b2g_trpo_upload_bytes(const b2g_trpo* h, int64_t* observe_bytes, int64_t* other_bytes) { return ac_upload_bytes(h, observe_bytes, other_bytes); }
int b2g_trpo_set_norm_stats(b2g_trpo* h, double clip_obs, double eps, int norm_obs) { B2G_TRPO_HANDLE(h); return ac_set_norm_stats(h, clip_obs, eps, norm_obs); }
int b2g_trpo_set_obs_encoder(b2g_trpo* h, const b2g_encoder* enc, int tail) { B2G_TRPO_HANDLE(h); return ac_set_obs_encoder(h, enc, tail); }
int b2g_trpo_observe_act(b2g_trpo* h, const float* obs, int n, int update_stats, float* act_out) {
  B2G_TRPO_HANDLE(h);
  return ac_observe_act(h, obs, n, update_stats, act_out, h->carried);
}
int b2g_trpo_act_raw(b2g_trpo* h, const float* obs, int n, int deterministic, float* act_out, float* value_out) {
  B2G_TRPO_HANDLE(h);
  if (!obs || !act_out || n < 0) return b2g_fail(B2G_EINVAL, "bad argument");
  return ac_predict(h, obs, n, deterministic, act_out, value_out, nullptr, true);
}
#undef B2G_TRPO_HANDLE

}  // extern "C"

// ================================================================================================
// Training state (b2g_trpo_state_save / _load; ac_state_save in actor_critic.cuh): the parameter arena holds pi and oldpi, the
// moments are the value Adam's.  The carried boundary action is not saved (every learn() starts from env.reset()).
// ================================================================================================
namespace {

std::vector<FpField> trpo_fingerprint(const b2g_trpo* h) {
  const b2g_trpo_cfg& c = h->cfg;
  return {fp_int("obs_dim", c.obs_dim), fp_int("n_actions", c.n_actions), fp_int("hidden0", c.hidden0), fp_int("hidden1", c.hidden1),
          fp_int("timesteps_per_batch", c.timesteps_per_batch), fp_int("seed", (int64_t)c.seed)};
}

}  // namespace

extern "C" {

int b2g_trpo_state_save(b2g_trpo* h, const char* path) {
  if (!h || !path) return b2g_fail(B2G_EINVAL, "NULL argument");
  B2G_USABLE(h);
  return ac_state_save(h, path, STATE_KIND_TRPO, trpo_fingerprint(h));
}

int b2g_trpo_state_load(b2g_trpo* h, const char* path) {
  if (!h || !path) return b2g_fail(B2G_EINVAL, "NULL argument");
  const int rc = ac_state_load(h, path, STATE_KIND_TRPO, trpo_fingerprint(h), "TRPO");
  if (rc == 0) h->carried = false;
  return rc;
}

}  // extern "C"

// ================================================================================================
// Debug read-back of the handle's device buffers (b2g_debug_trpo_tensor; layouts in b200grasp.h)
// ================================================================================================
namespace {

int find_trpo_tensor(const b2g_trpo* h, const char* name, AcDebugBuf& b) {
  if (ac_debug_base(h, h->RMAX, name, b)) return 0;
  const int64_t N = h->N, NF = h->NF, R = h->RMAX, A = h->A, H0 = h->H0, H1 = h->H1, n = h->n_train, V = kVfBatch;
  const int64_t np = std::max<int64_t>(1, (int64_t)h->cfg.vf_iters * N);
  const struct { const char* nm; const void* p; int64_t n; int eb; } t[] = {
      {"atarg", h->atarg, N, 4},     {"mu_old", h->mu_old, N * A, 4}, {"nlp_old", h->nlp_old, N, 4}, {"sdm", h->sdm, N * A, 4},
      {"sdls", h->sdls, N * A, 4},   {"u", h->u, NF * A, 4},          {"T0", h->T0, NF * H0, 4},      {"T1", h->T1, NF * H1, 4},
      {"dZ1", h->dZ1, R * H1, 4},    {"dZ0", h->dZ0, R * H0, 4},      {"X", h->X, n, 4},              {"Rv", h->Rv, n, 4},
      {"Pv", h->Pv, n, 4},           {"Zv", h->Zv, n, 4},             {"FS", h->FS, n, 4},            {"Gv", h->Gv, n, 4},
      {"part", h->part, kDotBlocks, 8}, {"amax", h->amax, kDotBlocks, 8}, {"lspart", h->lspart, kNcand * kLsBlocks * 2, 8},
      {"sc", h->sc, SC_N, 8},        {"met", h->met, TM_N, 4},
      {"cand", h->cand, kNcand * (H0 + H0 * H1 + H1 + H1 * A + 2 * A), 4},
      {"Y0c", h->Y0c, kNcand * N * H0, 4}, {"Y1c", h->Y1c, kNcand * N * H1, 4}, {"dZls", h->dZls, N * H0, 4},
      {"vZ0", h->vZ0, V * H0, 4},    {"vY0", h->vY0, V * H0, 4},      {"vY1", h->vY1, V * H1, 4},     {"vdZ1", h->vdZ1, V * H1, 4},
      {"vdZ0", h->vdZ0, V * H0, 4},  {"perm", h->perm, np, 4},        {"vrowoff", h->vrowoff, np, 4}};
  for (const auto& e : t)
    if (!strcmp(name, e.nm)) { b.p = e.p; b.numel = e.n; b.elem_bytes = e.eb; return 0; }
  return b2g_fail(B2G_EINVAL, std::string("unknown TRPO debug tensor: ") + name);
}

}  // namespace

extern "C" {

int b2g_debug_trpo_tensor_info(const b2g_trpo* h, const char* name, int64_t* numel, int32_t* elem_bytes) {
  B2G_USABLE(h);
  if (!h || !name) return b2g_fail(B2G_EINVAL, "NULL argument");
  AcDebugBuf b;
  if (int rc = find_trpo_tensor(h, name, b)) return rc;
  return ac_debug_info(b, numel, elem_bytes);
}

int b2g_debug_trpo_cg(b2g_trpo* h, const float* obs, const float* actions, const float* adv, int iters, float* prev) {
  B2G_USABLE(h);
  if (!h || !obs || !actions || !adv || !prev) return b2g_fail(B2G_EINVAL, "NULL argument");
  if (iters < 1 || iters > 64) return b2g_fail(B2G_EINVAL, "iters must be in [1, 64]");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  cudaStream_t s = h->stream;
  const size_t N = h->N, n = (size_t)h->n_train;
  if (int rc = ac_upload_rows(h, h->r_obs, obs, h->N)) return rc;
  CK(cudaMemcpyAsync(h->r_act, actions, N * h->A * sizeof(float), cudaMemcpyDefault, s));
  CK(cudaMemcpyAsync(h->r_adv, adv, N * sizeof(float), cudaMemcpyDefault, s));
  policy_grad_issue(h, s);
  for (int it = 0; it + 1 < iters; ++it) cg_iteration_issue(h, s);
  CK(cudaMemcpyAsync(prev, h->X, n * sizeof(float), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(prev + n, h->Rv, n * sizeof(float), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(prev + 2 * n, h->Pv, n * sizeof(float), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(prev + 3 * n, h->sc, SC_N * sizeof(double), cudaMemcpyDeviceToHost, s));
  cg_iteration_issue(h, s);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(s));
  h->t = 0;
  h->carried = false;
  h->acted = false;
  h->ob_n = 0;
  return 0;
}

int b2g_debug_trpo_tensor(b2g_trpo* h, const char* name, void* dst, size_t bytes) {
  B2G_USABLE(h);
  if (!h || !name || !dst) return b2g_fail(B2G_EINVAL, "NULL argument");
  AcDebugBuf b;
  if (int rc = find_trpo_tensor(h, name, b)) return rc;
  return ac_debug_read(h, b, name, dst, bytes);
}

}  // extern "C"
