// libb200grasp: dueling double DQN learner -- the `sb.DQN` branch of sb_helper.py:155-165 (stable-baselines 2.10.1 deepq).
//
// Network (deepq/policies.py FeedForwardPolicy, dueling=True, layers=[h0, h1], ReLU): two towers on the observation, each with
// its own first layer, action_value obs -> h0 -> h1 -> n and state_value obs -> h0 -> h1 -> 1, Q = V + (A - mean_n A).  The step
// (deepq/build_graph.py build_train, double_q=True, grad_norm_clipping=10) is restated in oracle/dqn_ref.py:
//   a* = argmax Q_online(s'),  y = r + gamma (1 - done) Q_target(s', a*),  td = Q(s, a) - y,  loss = mean_b w_b huber(td_b),
//   every gradient tensor clipped on its own to L2 norm 10 (tf.clip_by_norm), then TF1 Adam.
// All layers run on the fp32 gather-GEMM engine (gg_simt.cu) as grouped launches: three forward groups (each layer of both
// towers for the three evaluations online(s), online(s'), target(s')), one fused per-sample tail, three backward groups.
// Output-layer weights are held with their row stride padded to 4 floats (n = 1 for the value) so every operand row is 16-byte
// aligned; get/set repack to the zip layout.  The hard target copy is the caller's (b2g_dqn_update_target): stable-baselines
// decides it by the environment-step count, which the device never sees.  The replay gather normalises with the statistics of
// b2g_dqn_set_norm_stats (raw transitions are stored); the actor (b2g_dqn_act) takes observations as the network sees them, the
// VecNormalize wrapper's output, as stable-baselines' act and predict do.  The replay, normalisation, step, training-state and
// metrics-log plumbing is the QLearner base shared with BDQ (q_learner.cu).
// With device statistics (b2g_dqn_obs_rms_set) the learn loop's actor side runs here too, on the observe path BDQ shares
// (q_learner.cu): b2g_dqn_observe_act / _add stage each new frame once, merge it into VecNormalize's obs_rms, act
// epsilon-greedily on the device (Philox stream 3, dqn_explore_kernel) and commit the transitions into the replay.
#include <cuda_runtime.h>
#include <math.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/b200grasp.h"
#include "common.cuh"
#include "host.cuh"
#include "q_learner.cuh"

using namespace b2g;

namespace {

// metric slots (prep_kernel zeroes all MET_COUNT; optim_kernel accumulates the post-clip squared norm at MET_GN_PI)
constexpr int DMET_LOSS = 0, DMET_MEANQ = 1, DMET_ABSTD = 2, DMET_GN2 = 3, DMET_NCLIP = 4;
constexpr float kGradClip = 10.0f;    // dqn.py passes grad_norm_clipping=10 to build_train
constexpr int kClipThreads = 512;

struct DqnTailArgs {
  int B, n, NAS;               // batch, actions, padded action stride
  float gamma;
  const float* V[3];           // [B,4] value outputs of the 3 evaluations (col 0)
  const float* A[3];           // [B,NAS] advantages of the 3 evaluations
  const float* act; int act_stride;   // action indices (as floats) inside the obs rows
  const float* rew; const float* done; const float* weights;
  float* dA;                   // [B,NAS] gradient wrt the advantages
  float* dV;                   // [B,4]
  float* td;                   // [B]
  float* metrics;
};

__device__ __forceinline__ float row_mean(const float* a, int n) {
  float m = 0.f;
  for (int k = 0; k < n; ++k) m += a[k];
  return m / (float)n;
}

// first maximal index of Q_k = v + (a_k - mean) (tf.argmax over the dueling output)
__device__ __forceinline__ int q_argmax(const float* a, float v, float mean, int n) {
  int best = 0;
  float bv = v + (a[0] - mean);
  for (int k = 1; k < n; ++k) {
    const float q = v + (a[k] - mean);
    if (q > bv) { bv = q; best = k; }
  }
  return best;
}

// dueling aggregation, double-Q target, Huber loss with IS weights, the backward seeds dA / dV, td and the loss metrics
__global__ void dqn_tail_kernel(DqnTailArgs t) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  float loss_b = 0.f, q_b = 0.f, atd_b = 0.f;
  if (b < t.B) {
    const float invB = 1.0f / (float)t.B;
    const size_t ra = (size_t)b * t.NAS, rv = (size_t)b * 4;
    const float* a1 = t.A[1] + ra;                           // online net picks at s'
    const int best = q_argmax(a1, t.V[1][rv], row_mean(a1, t.n), t.n);
    const float* a2 = t.A[2] + ra;                           // target net evaluates
    const float qt = t.V[2][rv] + (a2[best] - row_mean(a2, t.n));
    const float y = t.rew[b] + t.gamma * (1.f - t.done[b]) * qt;
    const float* a0 = t.A[0] + ra;
    const int ai = (int)(t.act[(size_t)b * t.act_stride] + 0.5f);
    const float q = t.V[0][rv] + (a0[ai] - row_mean(a0, t.n));
    const float td = q - y;
    t.td[b] = td;
    const float w = t.weights ? t.weights[b] : 1.f;
    const float ad = fabsf(td);
    loss_b = w * (ad < 1.f ? 0.5f * td * td : ad - 0.5f) * invB;     // tf_util.huber_loss, delta 1
    q_b = q * invB;
    atd_b = ad * invB;
    const float dq = w * fminf(fmaxf(td, -1.f), 1.f) * invB;
    float* da = t.dA + ra;
    for (int k = 0; k < t.NAS; ++k) da[k] = k < t.n ? dq * ((k == ai ? 1.f : 0.f) - 1.f / (float)t.n) : 0.f;
    float* dvp = t.dV + rv;
    dvp[0] = dq; dvp[1] = dvp[2] = dvp[3] = 0.f;
  }
  for (int o = 16; o > 0; o >>= 1) {
    loss_b += __shfl_xor_sync(0xffffffffu, loss_b, o);
    q_b += __shfl_xor_sync(0xffffffffu, q_b, o);
    atd_b += __shfl_xor_sync(0xffffffffu, atd_b, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(t.metrics + DMET_LOSS, loss_b); atomicAdd(t.metrics + DMET_MEANQ, q_b); atomicAdd(t.metrics + DMET_ABSTD, atd_b);
  }
}

struct ClipJob { long long off; int count; };

// tf.clip_by_norm per variable: one CTA per online tensor, g <- g * clip / max(||g||_2, clip) in place.  Also the squared norm
// before clipping (summed over the tensors) and the number of tensors the clip scaled.
__global__ void __launch_bounds__(kClipThreads) dqn_clip_kernel(float* __restrict__ G, const ClipJob* __restrict__ jobs, float clip,
                                                                float* __restrict__ metrics) {
  const ClipJob job = jobs[blockIdx.x];
  float* g = G + job.off;
  float s = 0.f;
  for (int i = threadIdx.x; i < job.count; i += blockDim.x) s += g[i] * g[i];
  __shared__ float red[kClipThreads / 32];
  __shared__ float s_den;
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
    const float norm = sqrtf(tot);
    atomicAdd(metrics + DMET_GN2, tot);
    if (norm > clip) atomicAdd(metrics + DMET_NCLIP, 1.f);
    s_den = fmaxf(norm, clip);
  }
  __syncthreads();
  const float den = s_den;
  for (int i = threadIdx.x; i < job.count; i += blockDim.x) g[i] = g[i] * clip / den;
}

// greedy actions of the online net on `rows` evaluated rows, and optionally their Q rows [rows][n]
__global__ void dqn_act_kernel(const float* __restrict__ A, const float* __restrict__ V, int rows, int n, int NAS, int* __restrict__ out,
                               float* __restrict__ q_out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= rows) return;
  const float* a = A + (size_t)b * NAS;
  const float v = V[(size_t)b * 4], mean = row_mean(a, n);
  out[b] = q_argmax(a, v, mean, n);
  if (q_out)
    for (int k = 0; k < n; ++k) q_out[(size_t)b * n + k] = v + (a[k] - mean);
}
// The epsilon-greedy actor of b2g_dqn_observe_act on `rows` evaluated rows (env row0 + b): the greedy action of dqn_act_kernel
// and, with probability eps, a uniform random action instead.  Philox stream 3 at step counters[7] (the number of earlier
// acting observe_act calls), block row0 + b: lane x decides ((x + 0.5) 2^-32 < eps in float64, so eps = 0 never explores and
// eps = 1 always does), lane y picks the action (y * n) >> 32 -- bdq_explore_kernel's rule with one branch.  One CTA; the last
// chunk of a call advances the counter.
__global__ void dqn_explore_kernel(const float* __restrict__ A, const float* __restrict__ V, int rows, int row0, int n, int NAS, float eps,
                                   unsigned long long seed, long long* counters, int advance, int* __restrict__ out) {
  const unsigned long long step = (unsigned long long)counters[7];
  const uint2 key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  for (int b = threadIdx.x; b < rows; b += blockDim.x) {
    const float* a = A + (size_t)b * NAS;
    const int best = q_argmax(a, V[(size_t)b * 4], row_mean(a, n), n);
    const uint4 r = philox4x32_10(make_uint4((unsigned)step, (unsigned)(step >> 32), (unsigned)(row0 + b), 3u), key);
    const bool explore = ((double)r.x + 0.5) * (1.0 / 4294967296.0) < (double)eps;
    out[row0 + b] = explore ? (int)(((unsigned long long)r.y * (unsigned)n) >> 32) : best;
  }
  if (advance) {
    __syncthreads();
    if (threadIdx.x == 0) counters[7] = (long long)step + 1;
  }
}
}  // namespace

struct b2g_dqn : QLearner {     // A = 1
  b2g_dqn_cfg cfg{};
  int n = 0, NAS = 0, H0 = 0, H1 = 0;
  double* d_normc_act = nullptr;   // the actor's gather: observations arrive as the network sees them (no normalisation)
  float *h1[3][2]{}, *h2[3][2]{}, *Aout[3]{}, *Vout[3]{};      // [evaluation][tower 0 = action_value, 1 = state_value]
  float *dA = nullptr, *dV = nullptr, *dh2[2]{}, *dh1[2]{};
  float* q_rows = nullptr;
  ClipJob* clip_jobs = nullptr;
  int n_clip = 0;
};

namespace {
const char* const kTower[2] = {"action_value", "state_value"};
const std::string kOnline = "deepq/model", kTarget = "deepq/target_q_func/model";

std::string fcname(int i) { return i == 0 ? "fully_connected" : "fully_connected_" + std::to_string(i); }
std::string lname(int tw, int layer, const std::string& scope = kOnline) { return scope + "/" + kTower[tw] + "/" + fcname(layer); }

// an online tensor of the zip: weights [rows, cols] at row stride `stride`, biases [cols] padded to `stride`
void add_t(b2g_dqn* h, const std::string& name, int rows, int cols, bool w, int stride, int64_t& off) {
  h->params.add(name, w ? rows : 1, cols, w ? 2 : 1, stride, arena_take(off, w ? (int64_t)rows * stride : stride), true);
}

int build(b2g_dqn* h) {
  const int B = h->B, NAS = h->NAS, H0 = h->H0, H1 = h->H1, XS = h->XS, obs = h->E;
  const int *iH0, *iH1, *iNAS, *i4, *iobs, *rXS, *rH0, *rH1, *rNAS, *r4, *kH0, *kH1, *kNAS, *k4;
#define DT(var, vec) if (int rc = upload_table(h->allocs, h->stream, (vec), &var)) return rc;
  DT(iH0, iota_tab(H0)) DT(iH1, iota_tab(H1)) DT(iNAS, iota_tab(NAS)) DT(i4, iota_tab(4)) DT(iobs, iota_tab(XS))
  DT(rXS, iota_tab(B, XS)) DT(rH0, iota_tab(B, H0)) DT(rH1, iota_tab(B, H1)) DT(rNAS, iota_tab(B, NAS)) DT(r4, iota_tab(B, 4))
  DT(kH0, iota_tab(std::max(obs, H0) + 8, H0)) DT(kH1, iota_tab(std::max(H0, H1) + 8, H1)) DT(kNAS, iota_tab(H1 + 8, NAS))
  DT(k4, iota_tab(H1 + 8, 4))
#undef DT
  auto W = [&](int e, int tw, int layer, const char* wb) { return h->p(lname(tw, layer, e == 2 ? kTarget : kOnline) + wb); };
  // ---------------- forward: each layer of both towers for the 3 evaluations; the act groups hold evaluation 0 only
  for (int layer = 0; layer < 3; ++layer) {
    GemmGroup g, a;
    g.name = "dqn_fwd" + std::to_string(layer); a.name = "act_" + g.name;
    for (int e = 0; e < 3; ++e)
      for (int tw = 0; tw < 2; ++tw) {
        GemmDesc d;
        if (layer == 0)
          d = gemm_desc(e == 0 ? h->X : h->Xn, rXS, iobs, W(e, tw, 0, "/weights"), kH0, iH0, h->h1[e][tw], rH0, iH0, B, H0, obs,
                        GG_A_RVEC | GG_EPI_BIAS_RELU);
        else if (layer == 1)
          d = gemm_desc(h->h1[e][tw], rH0, iH0, W(e, tw, 1, "/weights"), kH1, iH1, h->h2[e][tw], rH1, iH1, B, H1, H0, GG_A_RVEC | GG_EPI_BIAS_RELU);
        else if (tw == 0)
          d = gemm_desc(h->h2[e][0], rH1, iH1, W(e, 0, 2, "/weights"), kNAS, iNAS, h->Aout[e], rNAS, iNAS, B, NAS, H1, GG_A_RVEC | GG_EPI_BIAS);
        else
          d = gemm_desc(h->h2[e][1], rH1, iH1, W(e, 1, 2, "/weights"), k4, i4, h->Vout[e], r4, i4, B, 4, H1, GG_A_RVEC | GG_EPI_BIAS);
        d.bias = W(e, tw, layer, "/biases");
        g.host.push_back(d);
        if (e == 0) a.host.push_back(d);
      }
    h->fwd.push_back(g); h->act.push_back(a);
  }
  // ---------------- backward (online evaluation 0), both towers per launch; no gradient into the observation
  {
    GemmGroup g; g.name = "dqn_out_bwd";
    for (int tw = 0; tw < 2; ++tw) {
      const int N = tw == 0 ? NAS : 4;
      const int *rN = tw == 0 ? rNAS : r4, *iN = tw == 0 ? iNAS : i4, *kN = tw == 0 ? kNAS : k4;
      const float* dz = tw == 0 ? h->dA : h->dV;
      GemmDesc w = gemm_desc(h->h2[0][tw], iH1, rH1, dz, rN, iN, h->g(lname(tw, 2) + "/weights"), kN, iN, H1, N, B, GG_COLSUM);
      w.colsum = h->g(lname(tw, 2) + "/biases");
      g.host.push_back(w);
      GemmDesc dg = gemm_desc(dz, rN, iN, h->p(lname(tw, 2) + "/weights"), iN, kN, h->dh2[tw], rH1, iH1, B, H1, N,
                              GG_A_RVEC | GG_B_RVEC | GG_EPI_MASK);
      dg.mask = h->h2[0][tw]; dg.kM = rH1; dg.kN = iH1;
      g.host.push_back(dg);
    }
    h->bwd.push_back(g);
  }
  {
    GemmGroup g; g.name = "dqn_hidden_bwd";
    for (int tw = 0; tw < 2; ++tw) {
      GemmDesc w = gemm_desc(h->h1[0][tw], iH0, rH0, h->dh2[tw], rH1, iH1, h->g(lname(tw, 1) + "/weights"), kH1, iH1, H0, H1, B, GG_COLSUM);
      w.colsum = h->g(lname(tw, 1) + "/biases");
      g.host.push_back(w);
      GemmDesc dg = gemm_desc(h->dh2[tw], rH1, iH1, h->p(lname(tw, 1) + "/weights"), iH1, kH1, h->dh1[tw], rH0, iH0, B, H0, H1,
                              GG_A_RVEC | GG_B_RVEC | GG_EPI_MASK);
      dg.mask = h->h1[0][tw]; dg.kM = rH0; dg.kN = iH0;
      g.host.push_back(dg);
    }
    h->bwd.push_back(g);
  }
  {
    GemmGroup g; g.name = "dqn_in_wgrad";
    for (int tw = 0; tw < 2; ++tw) {
      GemmDesc w = gemm_desc(h->X, iobs, rXS, h->dh1[tw], rH0, iH0, h->g(lname(tw, 0) + "/weights"), kH0, iH0, obs, H0, B, GG_COLSUM);
      w.colsum = h->g(lname(tw, 0) + "/biases");
      g.host.push_back(w);
    }
    h->bwd.push_back(g);
  }
  for (auto& g : h->fwd) if (int rc = finalize_tiles(g, h->allocs, h->stream)) return rc;
  for (auto& g : h->bwd) if (int rc = finalize_tiles(g, h->allocs, h->stream)) return rc;
  for (auto& g : h->act) if (int rc = finalize_tiles(g, h->allocs, h->stream)) return rc;
  // the clip jobs: every online tensor over its padded rows (pad columns hold zero gradients)
  std::vector<ClipJob> jobs;
  for (const ParamEntry& t : h->params.entries())
    if (t.grad) jobs.push_back(ClipJob{(long long)t.off, (int)(t.rows * t.stride)});
  h->n_clip = (int)jobs.size();
  if (int rc = dev_alloc(h->allocs, h->stream, &h->clip_jobs, jobs.size(), false)) return rc;
  CK(cudaMemcpyAsync(h->clip_jobs, jobs.data(), jobs.size() * sizeof(ClipJob), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}

int dqn_issue(b2g_dqn* h, bool sampled, bool apply, const float* weights) {
  cudaStream_t s = h->stream;
  PerArgs pr;
  if (int rc = ql_issue_prologue(h, sampled, apply, (size_t)h->n_train, &weights, &pr)) return rc;
  DqnTailArgs t{};
  t.B = h->B; t.n = h->n; t.NAS = h->NAS; t.gamma = h->gamma;
  for (int e = 0; e < 3; ++e) { t.V[e] = h->Vout[e]; t.A[e] = h->Aout[e]; }
  t.act = h->X + h->E; t.act_stride = h->XS;
  t.rew = h->rew_n; t.done = h->done_n; t.weights = weights;
  t.dA = h->dA; t.dV = h->dV; t.td = h->td; t.metrics = h->metrics;
  dqn_tail_kernel<<<(h->B + 127) / 128, 128, 0, s>>>(t);
  for (auto& g : h->bwd) gg_simt_launch(g.dev, (int)g.host.size(), g.total_tiles, s);
  dqn_clip_kernel<<<h->n_clip, kClipThreads, 0, s>>>(h->G, h->clip_jobs, kGradClip, h->metrics);
  ql_issue_priorities(h, sampled, pr);
  optim_launch(ql_optim_args(h, apply), s);
  if (apply && h->mlog.on()) {     // the dfetch accumulators (squared gradient norm, clip count as a float), the learning rate
    MetricsLogSrc m{};
    m.src[0] = h->metrics + DMET_LOSS; m.src[1] = h->metrics + DMET_MEANQ; m.src[2] = h->metrics + DMET_ABSTD;
    m.src[3] = h->metrics + DMET_GN2; m.src[4] = h->metrics + DMET_NCLIP; m.src[5] = h->d_lr;
    m.K = B2G_DQN_LOG_COLS;
    mlog_append(h->mlog, m, h->counters + 3, s);
  }
  CK(cudaGetLastError());
  return 0;
}

int dfetch(b2g_dqn* h, b2g_dqn_metrics* out) {
  if (int rc = ql_fetch(h)) return rc;
  if (out) {
    out->loss = h->h_met[DMET_LOSS]; out->mean_q = h->h_met[DMET_MEANQ]; out->mean_abs_td = h->h_met[DMET_ABSTD];
    out->grad_norm = sqrtf(h->h_met[DMET_GN2]); out->n_clipped = (int32_t)lrintf(h->h_met[DMET_NCLIP]);
    out->n_updates = h->n_updates;
  }
  return 0;
}
}  // namespace

extern "C" {

int b2g_dqn_destroy(b2g_dqn* h) {
  if (!h) return 0;
  ql_release(h);
  delete h;
  return 0;
}

int b2g_dqn_create(const b2g_dqn_cfg* cfg, b2g_dqn** out) { return b2g_dqn_create2(cfg, nullptr, out); }

int b2g_dqn_create2(const b2g_dqn_cfg* cfg, const b2g_replay_cfg* replay, b2g_dqn** out) {
  if (!cfg || !out) return b2g_fail(B2G_EINVAL, "cfg/out is NULL");
  *out = nullptr;
  if (cfg->n_actions < 2 || cfg->n_actions > 64) return b2g_fail(B2G_EINVAL, "n_actions must be in [2, 64]");
  if (cfg->hidden0 % 4 || cfg->hidden1 % 4 || cfg->hidden0 < 4 || cfg->hidden1 < 4 || cfg->hidden0 > 512 || cfg->hidden1 > 512)
    return b2g_fail(B2G_EINVAL, "hidden widths must be multiples of 4 in [4, 512]");
  if (cfg->obs_dim < 1 || cfg->batch < 1 || cfg->buffer_capacity < 1) return b2g_fail(B2G_EINVAL, "obs_dim, batch, buffer_capacity must be positive");
  if (cfg->prioritized_replay && cfg->batch > 1024) return b2g_fail(B2G_EINVAL, "prioritised replay supports batch <= 1024");
  if (cfg->batch > 65535) return b2g_fail(B2G_EINVAL, "batch must be <= 65535 (one gather CTA row per sample: grid.y)");
  if (int rc = check_replay_cfg(replay, cfg->buffer_capacity, 1)) return rc;
  if (int rc = check_device(cfg->device)) return rc;
  b2g_dqn* h = new b2g_dqn();
  h->cfg = *cfg;
  h->device = cfg->device; h->seed = cfg->seed; h->gamma = cfg->gamma;
  h->B = cfg->batch; h->E = cfg->obs_dim; h->XS = (cfg->obs_dim + 1 + 7) / 8 * 8;
  h->buffer_capacity = cfg->buffer_capacity; h->prioritized = cfg->prioritized_replay != 0;
  h->per_alpha = cfg->per_alpha; h->per_eps = cfg->per_eps;
  h->n = cfg->n_actions; h->NAS = (cfg->n_actions + 3) / 4 * 4;
  h->H0 = cfg->hidden0; h->H1 = cfg->hidden1;
  h->abi = "dqn";
  auto bail = [&](int rc) { std::string keep = g_b2g_err; b2g_dqn_destroy(h); g_b2g_err = keep; return rc; };
  // parameter inventory in zip order (oracle/dqn_ref.py all_specs)
  h->params.add_scalar("deepq/eps", &h->eps_value);
  int64_t off = 0;
  for (int tw = 0; tw < 2; ++tw) {
    const int no = tw == 0 ? h->n : 1, so = tw == 0 ? h->NAS : 4;
    add_t(h, lname(tw, 0) + "/weights", h->E, h->H0, true, h->H0, off);
    add_t(h, lname(tw, 0) + "/biases", 1, h->H0, false, h->H0, off);
    add_t(h, lname(tw, 1) + "/weights", h->H0, h->H1, true, h->H1, off);
    add_t(h, lname(tw, 1) + "/biases", 1, h->H1, false, h->H1, off);
    add_t(h, lname(tw, 2) + "/weights", h->H1, no, true, so, off);
    add_t(h, lname(tw, 2) + "/biases", 1, no, false, so, off);
  }
  h->n_train = off;
  h->params.add_copies(1, h->params.count() - 1, kOnline, kTarget, h->n_train);
  int rc = 0;
  const int B = h->B;
  if ((rc = ql_init(h, 0, replay, std::max(B, 256)))) return bail(rc);
  h->rms.set_call = "b2g_dqn_obs_rms_set";
#define DA(ptr, count) if ((rc = dev_alloc(h->allocs, h->stream, &(ptr), (size_t)(count)))) return bail(rc)
  DA(h->d_normc_act, 8);
  for (int e = 0; e < 3; ++e) {
    for (int tw = 0; tw < 2; ++tw) { DA(h->h1[e][tw], B * h->H0); DA(h->h2[e][tw], B * h->H1); }
    DA(h->Aout[e], B * h->NAS); DA(h->Vout[e], B * 4);
  }
  DA(h->dA, B * h->NAS); DA(h->dV, B * 4);
  for (int tw = 0; tw < 2; ++tw) { DA(h->dh2[tw], B * h->H1); DA(h->dh1[tw], B * h->H0); }
  DA(h->q_rows, B * h->n);
#undef DA
  {
    const double nc[8] = {1.0, 10.0, 10.0, 0.0, 0.0, 0, 0, 0};
    if (cudaMemcpyAsync(h->d_normc_act, nc, sizeof(nc), cudaMemcpyHostToDevice, h->stream) != cudaSuccess ||
        cudaStreamSynchronize(h->stream) != cudaSuccess)
      return bail(b2g_fail(B2G_ECUDA, "init copies"));
  }
  if ((rc = build(h))) return bail(rc);
  if (cudaStreamSynchronize(h->stream) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "create sync"));
  *out = h;
  return 0;
}

int b2g_dqn_param_count(const b2g_dqn* h) { return param_count(h); }
int b2g_dqn_param_info(const b2g_dqn* h, int idx, char* name, size_t name_cap, int64_t* rows, int64_t* cols, int32_t* ndim) {
  return param_info(h, idx, name, name_cap, rows, cols, ndim);
}
int b2g_dqn_get_param(b2g_dqn* h, const char* name, float* dst, size_t numel) { return param_copy(h, name, ParamCopy::Get, dst, numel); }
int b2g_dqn_set_param(b2g_dqn* h, const char* name, const float* src, size_t numel) {
  return param_copy(h, name, ParamCopy::Set, const_cast<float*>(src), numel);
}
int b2g_dqn_get_grad(b2g_dqn* h, const char* name, float* dst, size_t numel) { return param_copy(h, name, ParamCopy::GetGrad, dst, numel); }

// Every action must be an integer in [0, n_actions): the tail kernel indexes the Q row with it.  The values are read on the host
// (a device array is copied down first), before anything is stored or launched.
static int dqn_check_actions(const b2g_dqn* h, const float* act, int64_t n) {
  cudaPointerAttributes pa{};
  std::vector<float> tmp;
  const float* a = act;
  if (cudaPointerGetAttributes(&pa, act) == cudaSuccess && (pa.type == cudaMemoryTypeDevice)) {
    tmp.resize(n);
    CK(cudaMemcpy(tmp.data(), act, n * sizeof(float), cudaMemcpyDeviceToHost));
    a = tmp.data();
  }
  cudaGetLastError();      // a failed attribute query (the pointer is then host memory) leaves no error behind
  for (int64_t i = 0; i < n; ++i)
    if (!(a[i] >= 0.f && a[i] < (float)h->n && a[i] == floorf(a[i])))
      return b2g_fail(B2G_EINVAL, "action " + std::to_string(i) + " = " + std::to_string(a[i]) + " is not an integer in [0, " +
                                      std::to_string(h->n) + ")");
  return 0;
}

int b2g_dqn_replay_add(b2g_dqn* h, const float* obs, const float* act, const float* rew, const float* next_obs, const float* done, int64_t n) {
  if (int rc = ql_replay_add(h, obs, act, rew, next_obs, done, n, [&] { return dqn_check_actions(h, act, n); })) return rc;
  h->rms.up_other += (int64_t)(n * (2 * h->E + 3) * sizeof(float) + sizeof(long long));
  return 0;
}
int64_t b2g_dqn_replay_size(const b2g_dqn* h) { return ql_replay_size(h); }
int b2g_dqn_replay_info(const b2g_dqn* h, int64_t* capacity, int64_t* size, int64_t* frame_capacity, int64_t* live_frames, int64_t* bytes,
                        int64_t* evicted_early) {
  return ql_replay_info(h, capacity, size, frame_capacity, live_frames, bytes, evicted_early);
}
int b2g_dqn_replay_get(b2g_dqn* h, int64_t slot, float* obs, float* act, float* rew, float* next_obs, float* done, int32_t* frame_ids) {
  return ql_replay_get(h, slot, obs, act, rew, next_obs, done, frame_ids);
}
int b2g_dqn_set_norm_stats(b2g_dqn* h, const double* obs_mean, const double* obs_var, double ret_var, double clip_obs, double clip_rew, double eps,
                           int norm_obs, int norm_reward) {
  return ql_set_norm_stats(h, h ? &h->rms : nullptr, obs_mean, obs_var, ret_var, clip_obs, clip_rew, eps, norm_obs, norm_reward);
}
int b2g_dqn_step(b2g_dqn* h, int n_steps, float lr, b2g_dqn_metrics* out) {
  if (int rc = ql_step(h, n_steps, lr, [h] { return dqn_issue(h, true, true, nullptr); })) return rc;
  return dfetch(h, out);
}
int b2g_dqn_set_per_beta(b2g_dqn* h, float beta) { return ql_set_per_beta(h, beta); }
int b2g_dqn_get_last_per(b2g_dqn* h, int32_t* slots, float* weights, float* priorities) { return ql_get_last_per(h, slots, weights, priorities); }
int b2g_dqn_step_explicit(b2g_dqn* h, const float* obs, const float* act, const float* rew, const float* next_obs, const float* done,
                          const float* weights, float lr, int apply_update, b2g_dqn_metrics* out, float* td_out) {
  if (int rc = ql_step_explicit(h, obs, act, rew, next_obs, done, weights, lr, apply_update, td_out,
                                [&] { return dqn_check_actions(h, act, h->B); },
                                [h](bool apply, const float* w) { return dqn_issue(h, false, apply, w); }))
    return rc;
  return dfetch(h, out);
}

int b2g_dqn_update_target(b2g_dqn* h) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  CK(cudaSetDevice(h->device));
  CK(cudaMemcpyAsync(h->P + h->n_train, h->P, (size_t)h->n_train * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}

namespace {
// b2g_dqn_act (normc = the identity d_normc_act) and b2g_dqn_act_raw (normc = the gather's d_normc over obs_rms's table)
int dqn_act_rows(b2g_dqn* h, const float* obs, int n, int32_t* act_out, float* q_out, const double* normc) {
  CK(cudaSetDevice(h->device));
  const size_t E = h->E;
  for (int done_n = 0; done_n < n; done_n += h->B) {
    const int chunk = std::min(h->B, n - done_n);
    CK(cudaMemcpyAsync(h->s_obs, obs + (size_t)done_n * E, chunk * E * sizeof(float), cudaMemcpyDefault, h->stream));
    h->rms.up_other += (int64_t)(chunk * E * sizeof(float));
    GatherArgs g = ql_gather(h, false, false);
    g.normc = normc;
    gather_launch(g, h->stream);
    for (auto& gr : h->act) gg_simt_launch(gr.dev, (int)gr.host.size(), gr.total_tiles, h->stream);
    dqn_act_kernel<<<(chunk + 127) / 128, 128, 0, h->stream>>>(h->Aout[0], h->Vout[0], chunk, h->n, h->NAS, h->act_idx_out,
                                                               q_out ? h->q_rows : nullptr);
    CK(cudaMemcpyAsync(act_out + done_n, h->act_idx_out, chunk * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
    if (q_out)
      CK(cudaMemcpyAsync(q_out + (size_t)done_n * h->n, h->q_rows, (size_t)chunk * h->n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  CK(cudaGetLastError());
  return 0;
}
}  // namespace

int b2g_dqn_act(b2g_dqn* h, const float* obs, int n, int32_t* act_out, float* q_out) {
  B2G_USABLE(h);
  if (!h || !obs || !act_out || n < 0) return b2g_fail(B2G_EINVAL, "bad argument");
  return dqn_act_rows(h, obs, n, act_out, q_out, h->d_normc_act);
}

int b2g_dqn_act_raw(b2g_dqn* h, const float* obs, int n, int32_t* act_out, float* q_out) {
  B2G_USABLE(h);
  if (!h || !obs || !act_out || n < 0) return b2g_fail(B2G_EINVAL, "bad argument");
  if (!h->rms.on()) return b2g_fail(B2G_ESTATE, "act_raw normalises with the device statistics: call b2g_dqn_obs_rms_set first");
  return dqn_act_rows(h, obs, n, act_out, q_out, h->d_normc);
}

// ------------------------------------------------------------------------------------------------ obs_rms on the device and the
// actor loop fed from one upload per frame (the QLearner observe path, q_learner.cu; the templates of obsnorm.cuh read the
// QLearner view of device and nranks)
int b2g_dqn_obs_rms_set(b2g_dqn* h, const double* mean, const double* var, double count) {
  return obs_rms_set(static_cast<QLearner*>(h), mean, var, count);
}
int b2g_dqn_obs_rms_get(b2g_dqn* h, double* mean, double* var, double* count) { return obs_rms_get(static_cast<QLearner*>(h), mean, var, count); }
int b2g_dqn_upload_bytes(const b2g_dqn* h, int64_t* observe_bytes, int64_t* other_bytes) {
  return obs_rms_upload_bytes(static_cast<const QLearner*>(h), observe_bytes, other_bytes);
}

int b2g_dqn_set_obs_encoder(b2g_dqn* h, const b2g_encoder* enc, int tail) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  return ql_set_obs_encoder(h, enc, tail);
}

int b2g_dqn_observe_act(b2g_dqn* h, const float* obs, int n, int update_stats, float eps, int32_t* act_out) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  if (!obs && !act_out) return b2g_fail(B2G_EINVAL, "observe_act: nothing to do (obs and act_out are NULL)");
  if (act_out && !(eps >= 0.f && eps <= 1.f)) return b2g_fail(B2G_EINVAL, "observe_act: eps must be in [0, 1]");
  return ql_observe_act(h, obs, n, update_stats, act_out != nullptr, [&](const float* cur) {
    const unsigned long long seed = h->philox_key();
    for (int k = 0; k < n; k += h->B) {      // the act groups in chunks of batch rows, normalised with the gather's table
      const int chunk = std::min(h->B, n - k);
      GatherArgs g = ql_gather(h, false, false);
      g.obs = cur + (size_t)k * h->E;
      gather_launch(g, h->stream);
      for (auto& gr : h->act) gg_simt_launch(gr.dev, (int)gr.host.size(), gr.total_tiles, h->stream);
      dqn_explore_kernel<<<1, 256, 0, h->stream>>>(h->Aout[0], h->Vout[0], chunk, k, h->n, h->NAS, eps, seed, h->counters, k + chunk >= n,
                                                   h->ob_idx);
    }
    CK(cudaMemcpyAsync(act_out, h->ob_idx, n * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
    return 0;
  });
}

int b2g_dqn_observe_add(b2g_dqn* h, const float* act, const float* rew, const float* next_obs, const float* done, const float* reset_obs,
                        int n, int update_stats) {
  B2G_USABLE(h);
  if (!h || !act || !rew || !next_obs || !done) return b2g_fail(B2G_EINVAL, "NULL argument");
  return ql_observe_add(h, act, rew, next_obs, done, reset_obs, n, update_stats, [&] { return dqn_check_actions(h, act, n); });
}

}  // extern "C"

// ================================================================================================
// Training state (b2g_dqn_state_save / _load; container format in state.cuh)
// ================================================================================================
namespace {

std::vector<FpField> dqn_fingerprint(const b2g_dqn* h) {
  const b2g_dqn_cfg& c = h->cfg;
  return {fp_int("obs_dim", c.obs_dim), fp_int("n_actions", c.n_actions), fp_int("hidden0", c.hidden0), fp_int("hidden1", c.hidden1),
          fp_int("batch", c.batch), fp_int("buffer_capacity", c.buffer_capacity), fp_real("gamma", c.gamma), fp_int("seed", (int64_t)c.seed),
          fp_int("prioritized_replay", c.prioritized_replay), fp_real("per_alpha", c.per_alpha), fp_real("per_eps", c.per_eps)};
}

}  // namespace

extern "C" {

int b2g_dqn_state_save(b2g_dqn* h, const char* path) {
  return ql_state_save(h, path, STATE_KIND_DQN, h ? dqn_fingerprint(h) : std::vector<FpField>{}, h ? &h->rms : nullptr, nullptr);
}

int b2g_dqn_state_load(b2g_dqn* h, const char* path) {
  return ql_state_load(h, path, STATE_KIND_DQN, h ? dqn_fingerprint(h) : std::vector<FpField>{}, h ? &h->rms : nullptr, nullptr, "DQN",
                       [h] { h->ob_n = 0; });     // the staged observations are not part of the file: a fresh episode
}

int b2g_dqn_metrics_log(b2g_dqn* h, int capacity) { return ql_metrics_log(h, capacity, B2G_DQN_LOG_COLS); }

int b2g_dqn_metrics_drain(b2g_dqn* h, float* rows, int max_rows, int64_t* first_step, int* n_rows, int64_t* lost) {
  return ql_metrics_drain(h, rows, max_rows, first_step, n_rows, lost, [](float* r) {
    r[3] = sqrtf(r[3]); r[4] = (float)lrintf(r[4]);     // as dfetch
  });
}

}  // extern "C"
