// libb200grasp: branching dueling Q-network (BDQ) learner -- SURVEY.md section 8 row a11.
//
// The reference's BDQ lives in the absent `bdq_sb` fork (/root/reference/.gitmodules:1-3); call sites
// train_stable_baselines.py:103-104, sb_helper.py:202-226, hyper-parameters config/gripper_grasp.yaml:104-118.
// Algorithm restated in oracle/bdq_ref.py (Tavakoli et al., AAAI-18); variable names and shapes are the ones in
// trained_models/BDQ_8pads/BDQ_simple_8pads.zip.  PARITY UNPINNED (source absent).
//
// All layers are small dense contractions (<= 512 wide) and run on the fp32 gather-GEMM engine
// (gg_simt.cu) as grouped launches over the three network evaluations (online(s), online(s'), target(s'));
// the dueling aggregation, double-Q target, TD loss and backward seeds are one fused per-sample kernel.
// Output-layer weights are held with their row stride padded to 4 floats (n_bins = 33 -> 36) so every
// operand row is 16-byte aligned; get/set repack to the zip layout.
// The replay, normalisation, step, training-state and metrics-log plumbing is the QLearner base shared with DQN (q_learner.cu).
// With device statistics (b2g_bdq_obs_rms_set) the learn loop's actor side runs here too, on the observe path of the QLearner
// base (q_learner.cu, shared with DQN): b2g_bdq_observe_act / _add stage each new frame once, merge it into VecNormalize's
// obs_rms (ObsRms, obsnorm.cuh, shared with SAC), act epsilon-greedily on the device (Philox stream 3, bdq_explore_kernel) and
// commit transitions into the replay with a kernel.
#include <cuda_runtime.h>
#include <math.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/b200grasp.h"
#include "common.cuh"
#include "host.cuh"
#include "obsnorm.cuh"
#include "q_learner.cuh"

using namespace b2g;

namespace {

constexpr int BMET_LOSS = 0, BMET_MEANQ = 1, BMET_GN = MET_GN_PI;   // optim_kernel accumulates the squared norm at MET_GN_PI

struct BdqTailArgs {
  int B, D, n, NBS;            // batch, branches, bins, padded bin stride
  float gamma;
  const float* V[3];           // [B,4] value outputs of the 3 evaluations (col 0)
  const float* A[3][8];        // [B,NBS] advantages per evaluation / branch
  const float* act; int act_stride;   // action indices (as floats) inside the obs rows
  const float* rew; const float* done; const float* weights;
  float* dA[8];                // [B,NBS] gradient wrt advantages
  float* dV;                   // [B,4]
  float* td;                   // [B,D]
  float* metrics;
};

__global__ void bdq_tail_kernel(BdqTailArgs t) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  float loss_b = 0.f, q_b = 0.f;
  if (b < t.B) {
    const float invBD = 1.0f / (float)(t.B * t.D);
    float y = 0.f;
    for (int d = 0; d < t.D; ++d) {       // double-Q: online net picks, target net evaluates
      const float* a1 = t.A[1][d] + (size_t)b * t.NBS;
      int best = 0;
      float bv = a1[0];
      for (int k = 1; k < t.n; ++k) if (a1[k] > bv) { bv = a1[k]; best = k; }     // argmax_n (V + A - mean) = argmax_n A
      const float* a2 = t.A[2][d] + (size_t)b * t.NBS;
      float mean2 = 0.f;
      for (int k = 0; k < t.n; ++k) mean2 += a2[k];
      mean2 /= (float)t.n;
      y += t.V[2][(size_t)b * 4] + a2[best] - mean2;
    }
    y = t.rew[b] + t.gamma * (1.f - t.done[b]) * (y / (float)t.D);
    const float w = t.weights ? t.weights[b] : 1.f;
    float dv = 0.f;
    for (int d = 0; d < t.D; ++d) {
      const float* a0 = t.A[0][d] + (size_t)b * t.NBS;
      float mean0 = 0.f;
      for (int k = 0; k < t.n; ++k) mean0 += a0[k];
      mean0 /= (float)t.n;
      const int ai = (int)(t.act[(size_t)b * t.act_stride + d] + 0.5f);
      const float q = t.V[0][(size_t)b * 4] + a0[ai] - mean0;
      const float td = q - y;
      t.td[b * t.D + d] = td;
      loss_b += w * td * td;
      q_b += q;
      const float dq = 2.f * w * td * invBD;
      dv += dq;
      float* da = t.dA[d] + (size_t)b * t.NBS;
      for (int k = 0; k < t.NBS; ++k) da[k] = k < t.n ? dq * ((k == ai ? 1.f : 0.f) - 1.f / (float)t.n) : 0.f;
    }
    float* dvp = t.dV + (size_t)b * 4;
    dvp[0] = dv; dvp[1] = dvp[2] = dvp[3] = 0.f;
    loss_b *= invBD;
    q_b *= invBD;
  }
  for (int o = 16; o > 0; o >>= 1) {
    loss_b += __shfl_xor_sync(0xffffffffu, loss_b, o);
    q_b += __shfl_xor_sync(0xffffffffu, q_b, o);
  }
  if ((threadIdx.x & 31) == 0) { atomicAdd(t.metrics + BMET_LOSS, loss_b); atomicAdd(t.metrics + BMET_MEANQ, q_b); }
}

__global__ void bdq_argmax_kernel(const float* const* A, int n_rows, int D, int n, int NBS, int* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rows * D) return;
  const int b = i / D, d = i % D;
  const float* a = A[d] + (size_t)b * NBS;
  int best = 0;
  float bv = a[0];
  for (int k = 1; k < n; ++k) if (a[k] > bv) { bv = a[k]; best = k; }
  out[i] = best;
}

// The epsilon-greedy actor of b2g_bdq_observe_act on `rows` evaluated rows (env row0 + b): per branch the greedy bin, and with
// probability eps a uniform random bin instead, independently per (env, branch).  Philox stream 3 at step counters[7] (the
// number of earlier acting observe_act calls), block (row0 + b) * D + d: lane x decides, ((x + 0.5) 2^-32 < eps in float64, so
// eps = 0 never explores and eps = 1 always does), lane y picks the bin (y * n) >> 32.  One CTA; the last chunk of a call
// advances the counter.
__global__ void bdq_explore_kernel(const float* const* A, int rows, int row0, int D, int n, int NBS, float eps, unsigned long long seed,
                                   long long* counters, int advance, int* out) {
  const unsigned long long step = (unsigned long long)counters[7];
  const uint2 key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  for (int i = threadIdx.x; i < rows * D; i += blockDim.x) {
    const int b = i / D, d = i - b * D;
    const float* a = A[d] + (size_t)b * NBS;
    int best = 0;
    float bv = a[0];
    for (int k = 1; k < n; ++k) if (a[k] > bv) { bv = a[k]; best = k; }
    const unsigned blk = (unsigned)((row0 + b) * D + d);
    const uint4 r = philox4x32_10(make_uint4((unsigned)step, (unsigned)(step >> 32), blk, 3u), key);
    const bool explore = ((double)r.x + 0.5) * (1.0 / 4294967296.0) < (double)eps;
    out[(size_t)(row0 + b) * D + d] = explore ? (int)(((unsigned long long)r.y * (unsigned)n) >> 32) : best;
  }
  if (advance) {
    __syncthreads();
    if (threadIdx.x == 0) counters[7] = (long long)step + 1;
  }
}

// hard target copy every `freq` updates, decided on the device so that the step can live in a CUDA graph
__global__ void bdq_target_copy_kernel(float* __restrict__ P, long long n_train, const long long* __restrict__ counters, int freq) {
  if (freq <= 0 || counters[3] % freq != 0) return;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_train; i += (long long)gridDim.x * blockDim.x) P[n_train + i] = P[i];
}
}  // namespace

struct b2g_bdq : QLearner {     // A = D: one bin per branch
  b2g_bdq_cfg cfg{};
  int D = 0, n = 0, NBS = 0, T0 = 0, T1 = 0, HB = 0;
  float *h1[3]{}, *h2[3]{}, *hb[3][8]{}, *Aout[3][8]{}, *hv[3]{}, *Vout[3]{};
  float *dA[8]{}, *dV = nullptr, *dcat = nullptr, *dh2 = nullptr, *dh1 = nullptr;
  const float** d_Aptr = nullptr;
  void* nccl_comm = nullptr;
};

namespace {
std::string fcname(int i) { return i == 0 ? "fully_connected" : "fully_connected_" + std::to_string(i); }

// an online tensor of the zip: weights [rows, cols] at row stride `stride`, biases [cols] padded to `stride`
void add_t(b2g_bdq* h, const std::string& name, int rows, int cols, bool w, int stride, int64_t& off) {
  h->params.add(name, w ? rows : 1, cols, w ? 2 : 1, stride, arena_take(off, w ? (int64_t)rows * stride : stride), true);
}

int build(b2g_bdq* h) {
  const int B = h->B, D = h->D, NBS = h->NBS, T0 = h->T0, T1 = h->T1, HB = h->HB, XS = h->XS, obs = h->E;
  const int* iT0; const int* iT1; const int* iHB; const int* iNBS; const int* i4; const int* iobs;
  const int* rXS; const int* rT0; const int* rT1; const int* rHB; const int* rNBS; const int* r4; const int* rcat;
  const int* kT0; const int* kT1; const int* kHB; const int* kNBS; const int* k4; const int* icat;
#define BT(var, vec) if (int rc = upload_table(h->allocs, h->stream, (vec), &var)) return rc;
  BT(iT0, iota_tab(T0)) BT(iT1, iota_tab(T1)) BT(iHB, iota_tab(HB)) BT(iNBS, iota_tab(NBS)) BT(i4, iota_tab(4)) BT(iobs, iota_tab(XS))
  BT(rXS, iota_tab(B, XS)) BT(rT0, iota_tab(B, T0)) BT(rT1, iota_tab(B, T1)) BT(rHB, iota_tab(B, HB)) BT(rNBS, iota_tab(B, NBS)) BT(r4, iota_tab(B, 4))
  BT(rcat, iota_tab(B, (D + 1) * HB)) BT(icat, iota_tab((D + 1) * HB))
  BT(kT0, iota_tab(std::max(obs, T0) + 8, T0)) BT(kT1, iota_tab(std::max(T0, T1) + 8, T1)) BT(kHB, iota_tab(T1 + 8, HB)) BT(kNBS, iota_tab(HB + 8, NBS)) BT(k4, iota_tab(HB + 8, 4))
  const std::string sc[3] = {"bdq/model", "bdq/model", "bdq/target_q_func/model"};
  auto W = [&](int e, const std::string& rel) { return h->p((e == 2 ? "bdq/target_q_func/model" : "bdq/model") + rel); };
  // ---------------- forward (3 evaluations), also the policy-inference groups (evaluation 0 only)
  auto fwd_group = [&](const char* name, int layer) {
    GemmGroup g, a;
    g.name = name; a.name = std::string("act_") + name;
    for (int e = 0; e < 3; ++e) {
      const float* x = e == 0 ? h->X : h->Xn;
      std::vector<GemmDesc> ds;
      if (layer == 0) {
        GemmDesc d = gemm_desc(x, rXS, iobs, W(e, "/common_net/" + fcname(0) + "/weights"), kT0, iT0, h->h1[e], rT0, iT0, B, T0, obs, GG_A_RVEC | GG_EPI_BIAS_RELU);
        d.bias = W(e, "/common_net/" + fcname(0) + "/biases"); ds.push_back(d);
      } else if (layer == 1) {
        GemmDesc d = gemm_desc(h->h1[e], rT0, iT0, W(e, "/common_net/" + fcname(1) + "/weights"), kT1, iT1, h->h2[e], rT1, iT1, B, T1, T0, GG_A_RVEC | GG_EPI_BIAS_RELU);
        d.bias = W(e, "/common_net/" + fcname(1) + "/biases"); ds.push_back(d);
      } else if (layer == 2) {
        for (int q = 0; q <= D; ++q) {
          const std::string rel = q < D ? "/action_value/" + fcname(2 * q) : "/state_value/" + fcname(0);
          GemmDesc d = gemm_desc(h->h2[e], rT1, iT1, W(e, rel + "/weights"), kHB, iHB, q < D ? h->hb[e][q] : h->hv[e], rHB, iHB, B, HB, T1, GG_A_RVEC | GG_EPI_BIAS_RELU);
          d.bias = W(e, rel + "/biases"); ds.push_back(d);
        }
      } else {
        for (int q = 0; q <= D; ++q) {
          const std::string rel = q < D ? "/action_value/" + fcname(2 * q + 1) : "/state_value/" + fcname(1);
          const int N = q < D ? NBS : 4;
          GemmDesc d = gemm_desc(q < D ? h->hb[e][q] : h->hv[e], rHB, iHB, W(e, rel + "/weights"), q < D ? kNBS : k4, q < D ? iNBS : i4,
                           q < D ? h->Aout[e][q] : h->Vout[e], q < D ? rNBS : r4, q < D ? iNBS : i4, B, N, HB, GG_A_RVEC | GG_EPI_BIAS);
          d.bias = W(e, rel + "/biases"); ds.push_back(d);
        }
      }
      for (auto& d : ds) { g.host.push_back(d); if (e == 0) a.host.push_back(d); }
    }
    h->fwd.push_back(g); h->act.push_back(a);
  };
  fwd_group("bdq_trunk1", 0); fwd_group("bdq_trunk2", 1); fwd_group("bdq_hidden", 2); fwd_group("bdq_out", 3);
  // ---------------- backward (online evaluation 0)
  {
    GemmGroup g; g.name = "bdq_out_bwd";
    for (int q = 0; q <= D; ++q) {
      const std::string rel = q < D ? "bdq/model/action_value/" + fcname(2 * q + 1) : "bdq/model/state_value/" + fcname(1);
      const int N = q < D ? NBS : 4;
      const float* dz = q < D ? h->dA[q] : h->dV;
      const float* hin = q < D ? h->hb[0][q] : h->hv[0];
      GemmDesc w = gemm_desc(hin, iHB, rHB, dz, q < D ? rNBS : r4, q < D ? iNBS : i4, h->g(rel + "/weights"), q < D ? kNBS : k4, q < D ? iNBS : i4, HB, N, B, GG_COLSUM);
      w.colsum = h->g(rel + "/biases");
      g.host.push_back(w);
      // d(hidden) = (dz . W_out^T) masked by relu, written into the concatenated buffer [B, (D+1) HB] at column q HB
      const int* ccol; BT(ccol, iota_tab(HB, 1, q * HB))
      GemmDesc dg = gemm_desc(dz, q < D ? rNBS : r4, q < D ? iNBS : i4, h->p(rel + "/weights"), q < D ? iNBS : i4, q < D ? kNBS : k4, h->dcat, rcat, ccol, B, HB, N,
                        GG_A_RVEC | GG_B_RVEC | GG_EPI_MASK);
      dg.mask = hin; dg.kM = rHB; dg.kN = iHB;
      g.host.push_back(dg);
    }
    h->bwd.push_back(g);
  }
  {
    GemmGroup g; g.name = "bdq_hidden_bwd";
    std::vector<int> br((D + 1) * HB);
    for (int q = 0; q <= D; ++q) {
      const std::string rel = q < D ? "bdq/model/action_value/" + fcname(2 * q) : "bdq/model/state_value/" + fcname(0);
      const int* dzcol; BT(dzcol, iota_tab(B, (D + 1) * HB, q * HB))
      GemmDesc w = gemm_desc(h->h2[0], iT1, rT1, h->dcat, dzcol, iHB, h->g(rel + "/weights"), kHB, iHB, T1, HB, B, GG_COLSUM);
      w.colsum = h->g(rel + "/biases");
      g.host.push_back(w);
      for (int r = 0; r < HB; ++r) br[q * HB + r] = (int)h->params.off(rel + "/weights") + r;
    }
    const int* brt; BT(brt, br)
    GemmDesc dg = gemm_desc(h->dcat, rcat, icat, h->P, brt, kHB, h->dh2, rT1, iT1, B, T1, (D + 1) * HB, GG_A_RVEC | GG_B_RVEC | GG_EPI_MASK | GG_EPI_SCALE);
    dg.mask = h->h2[0]; dg.kM = rT1; dg.kN = iT1;
    dg.alpha = h->cfg.trunk_grad_rescale ? 1.0f / (float)(D + 1) : 1.0f;
    g.host.push_back(dg);
    h->bwd.push_back(g);
  }
  {
    GemmGroup g; g.name = "bdq_trunk2_bwd";
    GemmDesc w = gemm_desc(h->h1[0], iT0, rT0, h->dh2, rT1, iT1, h->g("bdq/model/common_net/" + fcname(1) + "/weights"), kT1, iT1, T0, T1, B, GG_COLSUM);
    w.colsum = h->g("bdq/model/common_net/" + fcname(1) + "/biases");
    g.host.push_back(w);
    GemmDesc dg = gemm_desc(h->dh2, rT1, iT1, h->p("bdq/model/common_net/" + fcname(1) + "/weights"), iT1, kT1, h->dh1, rT0, iT0, B, T0, T1, GG_A_RVEC | GG_B_RVEC | GG_EPI_MASK);
    dg.mask = h->h1[0]; dg.kM = rT0; dg.kN = iT0;
    g.host.push_back(dg);
    h->bwd.push_back(g);
  }
  {
    GemmGroup g; g.name = "bdq_trunk1_wgrad";
    GemmDesc w = gemm_desc(h->X, iobs, rXS, h->dh1, rT0, iT0, h->g("bdq/model/common_net/" + fcname(0) + "/weights"), kT0, iT0, obs, T0, B, GG_COLSUM);
    w.colsum = h->g("bdq/model/common_net/" + fcname(0) + "/biases");
    g.host.push_back(w);
    h->bwd.push_back(g);
  }
  for (auto& g : h->fwd) if (int rc = finalize_tiles(g, h->allocs, h->stream)) return rc;
  for (auto& g : h->bwd) if (int rc = finalize_tiles(g, h->allocs, h->stream)) return rc;
  for (auto& g : h->act) if (int rc = finalize_tiles(g, h->allocs, h->stream)) return rc;
  (void)sc;
  return 0;
}

int bdq_issue(b2g_bdq* h, bool sampled, bool apply, const float* weights) {
  cudaStream_t s = h->stream;
  PerArgs pr;
  if (int rc = ql_issue_prologue(h, sampled, apply, (size_t)(h->n_train + MET_COUNT), &weights, &pr)) return rc;
  BdqTailArgs t{};
  t.B = h->B; t.D = h->D; t.n = h->n; t.NBS = h->NBS; t.gamma = h->gamma;
  for (int e = 0; e < 3; ++e) { t.V[e] = h->Vout[e]; for (int d = 0; d < h->D; ++d) t.A[e][d] = h->Aout[e][d]; }
  t.act = h->X + h->E; t.act_stride = h->XS;
  t.rew = h->rew_n; t.done = h->done_n; t.weights = weights;
  for (int d = 0; d < h->D; ++d) t.dA[d] = h->dA[d];
  t.dV = h->dV; t.td = h->td; t.metrics = h->metrics;
  bdq_tail_kernel<<<(h->B + 127) / 128, 128, 0, s>>>(t);
  for (auto& g : h->bwd) gg_simt_launch(g.dev, (int)g.host.size(), g.total_tiles, s);
  ql_issue_priorities(h, sampled, pr);
  if (h->nranks > 1) {      // gradients + loss scalars averaged over the ranks (each rank sampled its own replay shard)
    CK(cudaMemcpyAsync(h->G + h->n_train, h->metrics, 2 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    if (int rc = nccl_allreduce_sum_f32(h->nccl_comm, h->G, (size_t)(h->n_train + MET_COUNT), s)) return rc;
    CK(cudaMemcpyAsync(h->metrics, h->G + h->n_train, 2 * sizeof(float), cudaMemcpyDeviceToDevice, s));
  }
  optim_launch(ql_optim_args(h, apply), s);
  CK(cudaGetLastError());
  if (apply) bdq_target_copy_kernel<<<64, 256, 0, s>>>(h->P, h->n_train, h->counters, h->cfg.target_update_freq);   // counters[3] = n_updates (prep)
  if (apply && h->mlog.on()) {     // loss and mean Q (sums over the ranks), the squared gradient norm, the learning rate
    MetricsLogSrc m{};
    m.src[0] = h->metrics + BMET_LOSS; m.src[1] = h->metrics + BMET_MEANQ; m.src[2] = h->metrics + BMET_GN; m.src[3] = h->d_lr;
    m.K = B2G_BDQ_LOG_COLS;
    mlog_append(h->mlog, m, h->counters + 3, s);
  }
  CK(cudaGetLastError());
  return 0;
}

int bfetch(b2g_bdq* h, b2g_bdq_metrics* out) {
  if (int rc = ql_fetch(h)) return rc;
  if (out) {
    const float inv = 1.0f / (float)h->nranks;
    out->loss = h->h_met[BMET_LOSS] * inv; out->mean_q = h->h_met[BMET_MEANQ] * inv; out->grad_norm = sqrtf(h->h_met[BMET_GN]);
    out->n_updates = h->n_updates;
  }
  return 0;
}
}  // namespace

extern "C" {

int b2g_bdq_destroy(b2g_bdq* h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  // the step graph first: with nranks > 1 it holds a captured all-reduce, whose resources NCCL reclaims through the communicator
  if (h->graph_exec) { cudaGraphExecDestroy(h->graph_exec); h->graph_exec = nullptr; }
  nccl_comm_destroy(h->nccl_comm);
  ql_release(h);
  delete h;
  return 0;
}

int b2g_bdq_create(const b2g_bdq_cfg* cfg, b2g_bdq** out) { return b2g_bdq_create2(cfg, nullptr, out); }

int b2g_bdq_create2(const b2g_bdq_cfg* cfg, const b2g_replay_cfg* replay, b2g_bdq** out) {
  if (!cfg || !out) return b2g_fail(B2G_EINVAL, "cfg/out is NULL");
  *out = nullptr;
  if (cfg->n_branches < 1 || cfg->n_branches > 8 || cfg->n_bins < 2 || cfg->n_bins > 64) return b2g_fail(B2G_EINVAL, "n_branches in [1,8], n_bins in [2,64]");
  if (cfg->trunk0 % 4 || cfg->trunk1 % 4 || cfg->branch_hidden % 4 || cfg->trunk0 < 4 || cfg->trunk1 < 4 || cfg->branch_hidden < 4)
    return b2g_fail(B2G_EINVAL, "layer widths must be positive multiples of 4");
  if (cfg->obs_dim < 1 || cfg->batch < 1 || cfg->buffer_capacity < 1) return b2g_fail(B2G_EINVAL, "obs_dim, batch, buffer_capacity must be positive");
  if (cfg->nranks < 1 || cfg->rank < 0 || cfg->rank >= cfg->nranks) return b2g_fail(B2G_EINVAL, "bad rank/nranks");
  if (cfg->nranks > 1 && !cfg->nccl_id) return b2g_fail(B2G_EINVAL, "nranks > 1 needs nccl_id");
  if (cfg->prioritized_replay && cfg->batch > 1024) return b2g_fail(B2G_EINVAL, "prioritised replay supports batch <= 1024");
  if (int rc = check_replay_cfg(replay, cfg->buffer_capacity, cfg->nranks)) return rc;
  if (int rc = check_device(cfg->device)) return rc;
  b2g_bdq* h = new b2g_bdq();
  h->cfg = *cfg;
  h->cfg.nccl_id = nullptr; h->cfg.nccl_lib = nullptr;
  h->device = cfg->device; h->rank = cfg->rank; h->nranks = cfg->nranks; h->seed = cfg->seed; h->gamma = cfg->gamma;
  h->B = cfg->batch; h->E = cfg->obs_dim; h->XS = (cfg->obs_dim + cfg->n_branches + 7) / 8 * 8; h->A = cfg->n_branches;
  h->buffer_capacity = cfg->buffer_capacity; h->prioritized = cfg->prioritized_replay != 0;
  h->per_alpha = cfg->per_alpha; h->per_eps = cfg->per_eps;
  h->D = cfg->n_branches; h->n = cfg->n_bins; h->NBS = (cfg->n_bins + 3) / 4 * 4;
  h->T0 = cfg->trunk0; h->T1 = cfg->trunk1; h->HB = cfg->branch_hidden;
  h->abi = "bdq";
  auto bail = [&](int rc) { std::string keep = g_b2g_err; b2g_bdq_destroy(h); g_b2g_err = keep; return rc; };
  // parameter inventory: same names and order as the zips (oracle/bdq_ref.py all_specs)
  h->params.add_scalar("bdq/eps", &h->eps_value);
  int64_t off = 0;
  for (int d = 0; d < h->D; ++d) {
    add_t(h, "bdq/model/action_value/" + fcname(2 * d) + "/biases", 1, h->HB, false, h->HB, off);
    add_t(h, "bdq/model/action_value/" + fcname(2 * d) + "/weights", h->T1, h->HB, true, h->HB, off);
    add_t(h, "bdq/model/action_value/" + fcname(2 * d + 1) + "/biases", 1, h->n, false, h->NBS, off);
    add_t(h, "bdq/model/action_value/" + fcname(2 * d + 1) + "/weights", h->HB, h->n, true, h->NBS, off);
  }
  add_t(h, "bdq/model/common_net/" + fcname(0) + "/biases", 1, h->T0, false, h->T0, off);
  add_t(h, "bdq/model/common_net/" + fcname(0) + "/weights", cfg->obs_dim, h->T0, true, h->T0, off);
  add_t(h, "bdq/model/common_net/" + fcname(1) + "/biases", 1, h->T1, false, h->T1, off);
  add_t(h, "bdq/model/common_net/" + fcname(1) + "/weights", h->T0, h->T1, true, h->T1, off);
  add_t(h, "bdq/model/state_value/" + fcname(0) + "/biases", 1, h->HB, false, h->HB, off);
  add_t(h, "bdq/model/state_value/" + fcname(0) + "/weights", h->T1, h->HB, true, h->HB, off);
  add_t(h, "bdq/model/state_value/" + fcname(1) + "/biases", 1, 1, false, 4, off);
  add_t(h, "bdq/model/state_value/" + fcname(1) + "/weights", h->HB, 1, true, 4, off);
  h->n_train = off;
  h->params.add_copies(1, h->params.count() - 1, "bdq/model", "bdq/target_q_func/model", h->n_train);
  int rc = 0;
  const int B = h->B, D = h->D;
  if ((rc = ql_init(h, MET_COUNT, replay, std::max(cfg->batch, 256)))) return bail(rc);     // the metrics ride the all-reduce in G
#define BA(ptr, count) if ((rc = dev_alloc(h->allocs, h->stream, &(ptr), (size_t)(count)))) return bail(rc)
  for (int e = 0; e < 3; ++e) {
    BA(h->h1[e], B * h->T0); BA(h->h2[e], B * h->T1); BA(h->hv[e], B * h->HB); BA(h->Vout[e], B * 4);
    for (int d = 0; d < D; ++d) { BA(h->hb[e][d], B * h->HB); BA(h->Aout[e][d], B * h->NBS); }
  }
  for (int d = 0; d < D; ++d) BA(h->dA[d], B * h->NBS);
  BA(h->dV, B * 4); BA(h->dcat, (size_t)B * (D + 1) * h->HB); BA(h->dh2, B * h->T1); BA(h->dh1, B * h->T0);
  BA(h->d_Aptr, 8);
#undef BA
  {
    const float* ap[8] = {};
    for (int d = 0; d < D; ++d) ap[d] = h->Aout[0][d];
    if (cudaMemcpyAsync(h->d_Aptr, ap, sizeof(ap), cudaMemcpyHostToDevice, h->stream) != cudaSuccess ||
        cudaStreamSynchronize(h->stream) != cudaSuccess)
      return bail(b2g_fail(B2G_ECUDA, "init copies"));
  }
  h->rms.set_call = "b2g_bdq_obs_rms_set";
  if ((rc = build(h))) return bail(rc);
  if (cfg->nranks > 1) {
    if ((rc = nccl_comm_init(&h->nccl_comm, cfg->nranks, cfg->nccl_id, cfg->rank, cfg->nccl_lib))) return bail(rc);
    if ((rc = nccl_allreduce_sum_f32(h->nccl_comm, h->G, (size_t)(h->n_train + MET_COUNT), h->stream))) return bail(rc);   // warm-up outside capture
  }
  if (cudaStreamSynchronize(h->stream) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "create sync"));
  *out = h;
  return 0;
}

int b2g_bdq_param_count(const b2g_bdq* h) { return param_count(h); }
int b2g_bdq_param_info(const b2g_bdq* h, int idx, char* name, size_t name_cap, int64_t* rows, int64_t* cols, int32_t* ndim) {
  return param_info(h, idx, name, name_cap, rows, cols, ndim);
}
int b2g_bdq_get_param(b2g_bdq* h, const char* name, float* dst, size_t numel) { return param_copy(h, name, ParamCopy::Get, dst, numel); }
int b2g_bdq_set_param(b2g_bdq* h, const char* name, const float* src, size_t numel) {
  return param_copy(h, name, ParamCopy::Set, const_cast<float*>(src), numel);
}
int b2g_bdq_get_grad(b2g_bdq* h, const char* name, float* dst, size_t numel) { return param_copy(h, name, ParamCopy::GetGrad, dst, numel); }

int b2g_bdq_replay_add(b2g_bdq* h, const float* obs, const float* act_idx, const float* rew, const float* next_obs, const float* done, int64_t n) {
  if (int rc = ql_replay_add(h, obs, act_idx, rew, next_obs, done, n, nullptr)) return rc;
  h->rms.up_other += (int64_t)(n * (2 * h->E + h->D + 2) * sizeof(float) + sizeof(long long));
  return 0;
}
int64_t b2g_bdq_replay_size(const b2g_bdq* h) { return ql_replay_size(h); }
int b2g_bdq_replay_info(const b2g_bdq* h, int64_t* capacity, int64_t* size, int64_t* frame_capacity, int64_t* live_frames, int64_t* bytes,
                        int64_t* evicted_early) {
  return ql_replay_info(h, capacity, size, frame_capacity, live_frames, bytes, evicted_early);
}
int b2g_bdq_replay_get(b2g_bdq* h, int64_t slot, float* obs, float* act_idx, float* rew, float* next_obs, float* done, int32_t* frame_ids) {
  return ql_replay_get(h, slot, obs, act_idx, rew, next_obs, done, frame_ids);
}
int b2g_bdq_set_norm_stats(b2g_bdq* h, const double* obs_mean, const double* obs_var, double ret_var, double clip_obs, double clip_rew, double eps,
                           int norm_obs, int norm_reward) {
  return ql_set_norm_stats(h, h ? &h->rms : nullptr, obs_mean, obs_var, ret_var, clip_obs, clip_rew, eps, norm_obs, norm_reward);
}
int b2g_bdq_step(b2g_bdq* h, int n_steps, float lr, b2g_bdq_metrics* out) {
  if (int rc = ql_step(h, n_steps, lr, [h] { return bdq_issue(h, true, true, nullptr); })) return rc;
  return bfetch(h, out);
}
int b2g_bdq_set_per_beta(b2g_bdq* h, float beta) { return ql_set_per_beta(h, beta); }
int b2g_bdq_get_last_per(b2g_bdq* h, int32_t* slots, float* weights, float* priorities) { return ql_get_last_per(h, slots, weights, priorities); }
int b2g_bdq_step_explicit(b2g_bdq* h, const float* obs, const float* act_idx, const float* rew, const float* next_obs, const float* done,
                          const float* weights, float lr, int apply_update, b2g_bdq_metrics* out, float* td_out) {
  if (int rc = ql_step_explicit(h, obs, act_idx, rew, next_obs, done, weights, lr, apply_update, td_out, nullptr,
                                [h](bool apply, const float* w) { return bdq_issue(h, false, apply, w); }))
    return rc;
  return bfetch(h, out);
}

// greedy branch actions argmax_n Q_d(s, n) of the online network (the epsilon-greedy mixing is the caller's)
int b2g_bdq_act(b2g_bdq* h, const float* obs, int n, int32_t* act_idx_out) {
  B2G_USABLE(h);
  if (!h || !obs || !act_idx_out || n < 0) return b2g_fail(B2G_EINVAL, "bad argument");
  CK(cudaSetDevice(h->device));
  const size_t E = h->E, D = h->D;
  for (int done_n = 0; done_n < n; done_n += h->B) {
    const int chunk = std::min(h->B, n - done_n);
    CK(cudaMemcpyAsync(h->s_obs, obs + (size_t)done_n * E, chunk * E * sizeof(float), cudaMemcpyDefault, h->stream));
    h->rms.up_other += (int64_t)(chunk * E * sizeof(float));
    GatherArgs g = ql_gather(h, false, false);
    gather_launch(g, h->stream);
    for (auto& gr : h->act) gg_simt_launch(gr.dev, (int)gr.host.size(), gr.total_tiles, h->stream);
    bdq_argmax_kernel<<<(chunk * (int)D + 127) / 128, 128, 0, h->stream>>>(h->d_Aptr, chunk, (int)D, h->n, h->NBS, h->act_idx_out);
    CK(cudaMemcpyAsync(act_idx_out + (size_t)done_n * D, h->act_idx_out, chunk * D * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  CK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------ obs_rms on the device and the
// actor loop fed from one upload per frame (ObsRms, obsnorm.cuh; the merge is obsnorm.cu's kernel over the flat layout)
int b2g_bdq_obs_rms_set(b2g_bdq* h, const double* mean, const double* var, double count) { return obs_rms_set(h, mean, var, count); }
int b2g_bdq_obs_rms_get(b2g_bdq* h, double* mean, double* var, double* count) { return obs_rms_get(h, mean, var, count); }
int b2g_bdq_upload_bytes(const b2g_bdq* h, int64_t* observe_bytes, int64_t* other_bytes) {
  return obs_rms_upload_bytes(h, observe_bytes, other_bytes);
}

int b2g_bdq_set_obs_encoder(b2g_bdq* h, const b2g_encoder* enc, int tail) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  return ql_set_obs_encoder(h, enc, tail);
}

int b2g_bdq_observe_act(b2g_bdq* h, const float* obs, int n, int update_stats, float eps, int32_t* act_idx_out) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  if (!obs && !act_idx_out) return b2g_fail(B2G_EINVAL, "observe_act: nothing to do (obs and act_idx_out are NULL)");
  if (act_idx_out && !(eps >= 0.f && eps <= 1.f)) return b2g_fail(B2G_EINVAL, "observe_act: eps must be in [0, 1]");
  return ql_observe_act(h, obs, n, update_stats, act_idx_out != nullptr, [&](const float* cur) {
    const size_t E = h->E, D = h->D;
    const unsigned long long seed = h->philox_key();
    for (int k = 0; k < n; k += h->B) {
      const int chunk = std::min(h->B, n - k);
      GatherArgs g = ql_gather(h, false, false);
      g.obs = cur + (size_t)k * E;
      gather_launch(g, h->stream);
      for (auto& gr : h->act) gg_simt_launch(gr.dev, (int)gr.host.size(), gr.total_tiles, h->stream);
      bdq_explore_kernel<<<1, 256, 0, h->stream>>>(h->d_Aptr, chunk, k, (int)D, h->n, h->NBS, eps, seed, h->counters, k + chunk >= n, h->ob_idx);
    }
    CK(cudaMemcpyAsync(act_idx_out, h->ob_idx, n * D * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
    return 0;
  });
}

int b2g_bdq_observe_add(b2g_bdq* h, const float* act_idx, const float* rew, const float* next_obs, const float* done, const float* reset_obs,
                        int n, int update_stats) {
  B2G_USABLE(h);
  if (!h || !act_idx || !rew || !next_obs || !done) return b2g_fail(B2G_EINVAL, "NULL argument");
  return ql_observe_add(h, act_idx, rew, next_obs, done, reset_obs, n, update_stats, nullptr);
}

}  // extern "C"

// ================================================================================================
// Training state (b2g_bdq_state_save / _load; container format in state.cuh)
// ================================================================================================
namespace {

std::vector<FpField> bdq_fingerprint(const b2g_bdq* h) {
  const b2g_bdq_cfg& c = h->cfg;
  return {fp_int("obs_dim", c.obs_dim), fp_int("n_branches", c.n_branches), fp_int("n_bins", c.n_bins), fp_int("trunk0", c.trunk0),
          fp_int("trunk1", c.trunk1), fp_int("branch_hidden", c.branch_hidden), fp_int("batch", c.batch),
          fp_int("buffer_capacity", c.buffer_capacity), fp_real("gamma", c.gamma), fp_int("target_update_freq", c.target_update_freq),
          fp_int("trunk_grad_rescale", c.trunk_grad_rescale), fp_int("seed", (int64_t)c.seed),
          fp_int("prioritized_replay", c.prioritized_replay), fp_real("per_alpha", c.per_alpha), fp_real("per_eps", c.per_eps)};
}
}  // namespace

extern "C" {

int b2g_bdq_state_save(b2g_bdq* h, const char* path) {
  return ql_state_save(h, path, STATE_KIND_BDQ, h ? bdq_fingerprint(h) : std::vector<FpField>{}, h ? &h->rms : nullptr,
                       h && h->nranks > 1 ? "training-state files of data-parallel learners (nranks > 1) are not built: each rank "
                                                "holds its own replay shard"
                                              : nullptr);
}

int b2g_bdq_state_load(b2g_bdq* h, const char* path) {
  return ql_state_load(h, path, STATE_KIND_BDQ, h ? bdq_fingerprint(h) : std::vector<FpField>{}, h ? &h->rms : nullptr,
                       h && h->nranks > 1 ? "training-state files of data-parallel learners (nranks > 1) are not built" : nullptr,
                       "BDQ", [h] { h->ob_n = 0; });     // the staged observations are not part of the file: a fresh episode
}

int b2g_bdq_metrics_log(b2g_bdq* h, int capacity) { return ql_metrics_log(h, capacity, B2G_BDQ_LOG_COLS); }

int b2g_bdq_metrics_drain(b2g_bdq* h, float* rows, int max_rows, int64_t* first_step, int* n_rows, int64_t* lost) {
  const float inv = h ? 1.0f / (float)h->nranks : 1.0f;
  return ql_metrics_drain(h, rows, max_rows, first_step, n_rows, lost, [inv](float* r) {
    r[0] *= inv; r[1] *= inv; r[2] = sqrtf(r[2]);     // as bfetch
  });
}

}  // extern "C"
