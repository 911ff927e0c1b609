// The replay Q-learner shared by the BDQ and DQN handles (q_learner.cuh).
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "obsnorm.cuh"
#include "q_learner.cuh"

namespace b2g {

namespace {
// observe_add without frames: transition i = (cur[i], act[i][A], rew[i], nxt[i], done[i]) -> replay slot (first + i) % cap, one
// CTA per row; CTA 0 also writes the new replay size into counters[5] (what replay_add uploads)
__global__ void ql_commit_kernel(const float* __restrict__ cur, const float* __restrict__ nxt, const float* __restrict__ act,
                                 const float* __restrict__ rew, const float* __restrict__ done, int E, int A, long long first, long long cap,
                                 float* __restrict__ r_obs, float* __restrict__ r_next, float* __restrict__ r_act, float* __restrict__ r_rew,
                                 float* __restrict__ r_done, long long* counters, long long new_size) {
  const int i = blockIdx.x;
  const long long slot = (first + i) % cap;
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    r_obs[slot * E + e] = cur[(size_t)i * E + e];
    r_next[slot * E + e] = nxt[(size_t)i * E + e];
  }
  if (threadIdx.x < A) r_act[slot * A + threadIdx.x] = act[(size_t)i * A + threadIdx.x];
  if (threadIdx.x == 0) { r_rew[slot] = rew[i]; r_done[slot] = done[i]; }
  if (i == 0 && threadIdx.x == 0) counters[5] = new_size;
}
}  // namespace

int ql_init(QLearner* h, int64_t g_extra, const b2g_replay_cfg* replay, int stage_rows) {
  const char* ng = getenv("B2G_NO_GRAPH");
  h->use_graph = !(ng && ng[0] == '1');
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) return b2g_fail(B2G_ECUDA, "stream");
  const int B = h->B, E = h->E, A = h->A;
#define QA(ptr, count) if (int rc = dev_alloc(h->allocs, h->stream, &(ptr), (size_t)(count))) return rc
  QA(h->P, 2 * h->n_train); QA(h->Mo, h->n_train); QA(h->Vo, h->n_train); QA(h->G, h->n_train + g_extra); QA(h->metrics, MET_COUNT);
  QA(h->counters, 8); QA(h->step_consts, 4); QA(h->d_lr, 1);
  if (int rc = h->replay.init(h->allocs, h->stream, h->buffer_capacity, E, A, B, h->prioritized, h->per_alpha, h->per_eps,
                              replay ? replay->frame_capacity : 0, plain_frames(E), stage_rows))
    return rc;
  QA(h->d_mean, E); QA(h->d_istd, E); QA(h->d_normc, 8);
  QA(h->X, (size_t)B * h->XS); QA(h->Xn, (size_t)B * h->XS); QA(h->Xscratch, (size_t)B * h->XS);
  QA(h->td, B * A);
  QA(h->rew_n, B); QA(h->done_n, B); QA(h->weights, B); QA(h->eps_dummy, B + 8); QA(h->indices, B + 4); QA(h->act_idx_out, B * A);
  QA(h->s_obs, (size_t)B * E); QA(h->s_next, (size_t)B * E); QA(h->s_act, B * A); QA(h->s_rew, B); QA(h->s_done, B);
#undef QA
  if (cudaMallocHost((void**)&h->h_met, MET_COUNT * sizeof(float)) != cudaSuccess) return b2g_fail(B2G_ECUDA, "cudaMallocHost");
  h->cfg.device = h->device; h->cfg.nranks = h->nranks;
  h->stage_rows = stage_rows;
  h->rms.E = E; h->rms.d_mean = h->d_mean; h->rms.d_istd = h->d_istd;
  std::vector<double> ones(E, 1.0);
  const double nc[8] = {1.0, 10.0, 10.0, 0.0, 0.0, 0, 0, 0};
  if (cudaMemcpyAsync(h->d_istd, ones.data(), E * sizeof(double), cudaMemcpyHostToDevice, h->stream) != cudaSuccess ||
      cudaMemcpyAsync(h->d_normc, nc, sizeof(nc), cudaMemcpyHostToDevice, h->stream) != cudaSuccess ||
      cudaStreamSynchronize(h->stream) != cudaSuccess)
    return b2g_fail(B2G_ECUDA, "init copies");
  return 0;
}

void ql_release(QLearner* h) {
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->graph_exec) cudaGraphExecDestroy(h->graph_exec);
  enc_stage_destroy(h->rms.enc);
  h->rms.enc = nullptr;
  mlog_free(&h->mlog);
  for (void* q : h->allocs) cudaFree(q);
  h->replay.release();
  if (h->h_met) cudaFreeHost(h->h_met);
  if (h->stream) cudaStreamDestroy(h->stream);
}

GatherArgs ql_gather(QLearner* h, bool from_replay, bool with_next) {
  GatherArgs g{};
  g.obs = h->s_obs; g.next_obs = with_next ? h->s_next : nullptr;
  g.act = with_next ? h->s_act : nullptr; g.rew = h->s_rew; g.done = h->s_done;
  if (from_replay) {
    h->replay.gather_args(g, with_next);
    g.indices = h->indices;
  }
  g.mean = h->d_mean; g.var = h->d_istd; g.normc = h->d_normc;
  g.B = h->B; g.H = 0; g.W = h->E; g.Cimg = 0; g.scale = 1.f;
  g.F_pi = h->Xscratch; g.F_v = h->X; g.F_t = h->Xn; g.FS = h->XS; g.feat_col = 0;
  g.rew_out = h->rew_n; g.done_out = h->done_n; g.n_act = h->A;
  return g;
}

int ql_issue_prologue(QLearner* h, bool sampled, bool apply, size_t g_floats, const float** weights, PerArgs* pr) {
  cudaStream_t s = h->stream;
  PrepArgs pa{};
  pa.counters = h->counters; pa.step_consts = h->step_consts; pa.lr = h->d_lr; pa.metrics = h->metrics;
  pa.indices = h->indices; pa.eps = h->eps_dummy; pa.B = h->B; pa.A = 1; pa.replay_size = nullptr;
  pa.seed = h->philox_key(); pa.gen = sampled ? 1 : 0; pa.apply = apply ? 1 : 0;
  pa.ring_cap = h->replay.ring_cap();
  prep_launch(pa, s);
  *pr = h->replay.per_args(h->counters, pa.seed, h->B, h->indices, h->weights, h->td, h->A);
  if (h->replay.per && sampled) { per_sample_launch(*pr, s); *weights = h->weights; }   // overwrites the uniform draw
  gather_launch(ql_gather(h, sampled, true), s);
  CK(cudaMemsetAsync(h->G, 0, g_floats * sizeof(float), s));
  for (auto& g : h->fwd) gg_simt_launch(g.dev, (int)g.host.size(), g.total_tiles, s);
  return 0;
}

void ql_issue_priorities(QLearner* h, bool sampled, const PerArgs& pr) {
  if (h->replay.per && sampled) per_write_launch(pr, h->indices, 0, h->buffer_capacity, h->B, 1, h->stream);
}

OptimArgs ql_optim_args(QLearner* h, bool apply) {
  OptimArgs oa{};
  oa.P = h->P; oa.Mo = h->Mo; oa.Vo = h->Vo; oa.G = h->G; oa.T = h->P + h->n_train;
  oa.n_pi = (int)h->n_train; oa.n_values = 0; oa.n_ent = 0; oa.n_target = 0;
  oa.step_consts = h->step_consts; oa.tau = 0.f; oa.grad_scale = 1.0f / (float)h->nranks; oa.metrics = h->metrics; oa.apply = apply ? 1 : 0;
  return oa;
}

int ql_fetch(QLearner* h) {
  CK(cudaMemcpyAsync(h->h_met, h->metrics, MET_COUNT * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------- entry points
int ql_replay_add(QLearner* h, const float* obs, const float* act, const float* rew, const float* next_obs, const float* done, int64_t n,
                  const std::function<int()>& check) {
  B2G_USABLE(h);
  if (!h || !obs || !act || !rew || !next_obs || !done || n < 0) return b2g_fail(B2G_EINVAL, "NULL argument");
  CK(cudaSetDevice(h->device));
  if (check)
    if (int rc = check()) return rc;
  return h->replay.add(obs, act, rew, next_obs, done, n, h->counters, h->stream);
}

int64_t ql_replay_size(const QLearner* h) { B2G_USABLE(h); return h ? h->replay.size : 0; }

int ql_replay_info(const QLearner* h, int64_t* capacity, int64_t* size, int64_t* frame_capacity, int64_t* live_frames, int64_t* bytes,
                   int64_t* evicted_early) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  h->replay.info(capacity, size, frame_capacity, live_frames, bytes, evicted_early);
  return 0;
}

int ql_replay_get(QLearner* h, int64_t slot, float* obs, float* act, float* rew, float* next_obs, float* done, int32_t* frame_ids) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  return h->replay.get(slot, obs, act, rew, next_obs, done, frame_ids, h->device, h->stream);
}

int ql_set_norm_stats(QLearner* h, ObsRms* rms, const double* obs_mean, const double* obs_var, double ret_var, double clip_obs,
                      double clip_rew, double eps, int norm_obs, int norm_reward) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  const bool own = rms && rms->on();
  if (norm_obs && !own && (!obs_mean || !obs_var)) return b2g_fail(B2G_EINVAL, "norm_obs needs obs_mean/obs_var");
  CK(cudaSetDevice(h->device));
  CK(cudaStreamSynchronize(h->stream));
  int64_t up = 0;
  if (rms)
    if (int rc = rms->norm_stats(obs_mean, obs_var, eps, h->device, h->nranks, h->allocs, h->stream)) return rc;
  if (!own && norm_obs) {
    std::vector<double> istd(h->E);
    for (int i = 0; i < h->E; ++i) istd[i] = 1.0 / sqrt(obs_var[i] + eps);
    CK(cudaMemcpy(h->d_mean, obs_mean, h->E * sizeof(double), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(h->d_istd, istd.data(), h->E * sizeof(double), cudaMemcpyHostToDevice));
    up += (int64_t)(2 * h->E * sizeof(double));
  }
  const double nc[8] = {1.0 / sqrt(ret_var + eps), clip_obs, clip_rew, (double)norm_obs, (double)norm_reward, 0, 0, 0};
  CK(cudaMemcpy(h->d_normc, nc, sizeof(nc), cudaMemcpyHostToDevice));
  if (rms) rms->up_other += up + (int64_t)sizeof(nc);
  return 0;
}

int ql_set_per_beta(QLearner* h, float beta) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  return h->replay.set_beta(beta, h->device, h->stream);
}

// h->indices holds the slots of the last sampled step with uniform replay too (prep_kernel draws them, per_sample_kernel
// overwrites them with PER); weights and prio_out are written by PER steps only
int ql_get_last_per(QLearner* h, int32_t* slots, float* weights, float* priorities) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  return h->replay.get_last(h->indices, h->weights, h->B, slots, weights, priorities, h->device, h->stream);
}

int ql_step(QLearner* h, int n_steps, float lr, const std::function<int()>& issue) {
  B2G_USABLE(h);
  if (!h || n_steps < 0) return b2g_fail(B2G_EINVAL, "bad argument");
  if (h->replay.size < 1) return b2g_fail(B2G_ESTATE, "replay buffer is empty");
  CK(cudaSetDevice(h->device));
  if (int rc = upload_lr(h->d_lr, &h->cur_lr, lr, h->stream)) return rc;
  if (h->use_graph && !h->graph_exec)       // the whole step (~14 launches of tiny layers) replays as one graph
    if (int rc = capture_graph(h->stream, issue, &h->graph_exec)) return rc;
  for (int i = 0; i < n_steps; ++i) {
    if (h->graph_exec) CK(cudaGraphLaunch(h->graph_exec, h->stream));
    else if (int rc = issue()) return rc;
    ++h->n_updates;
  }
  return 0;
}

int ql_step_explicit(QLearner* h, const float* obs, const float* act, const float* rew, const float* next_obs, const float* done,
                     const float* weights, float lr, int apply_update, float* td_out, const std::function<int()>& check,
                     const std::function<int(bool, const float*)>& issue) {
  B2G_USABLE(h);
  if (!h || !obs || !act || !rew || !next_obs || !done) return b2g_fail(B2G_EINVAL, "NULL argument");
  CK(cudaSetDevice(h->device));
  if (check)
    if (int rc = check()) return rc;
  if (int rc = upload_lr(h->d_lr, &h->cur_lr, lr, h->stream)) return rc;
  const size_t B = h->B, E = h->E, A = h->A;
  CK(cudaMemcpyAsync(h->s_obs, obs, B * E * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaMemcpyAsync(h->s_next, next_obs, B * E * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaMemcpyAsync(h->s_act, act, B * A * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaMemcpyAsync(h->s_rew, rew, B * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaMemcpyAsync(h->s_done, done, B * sizeof(float), cudaMemcpyDefault, h->stream));
  if (weights) CK(cudaMemcpyAsync(h->weights, weights, B * sizeof(float), cudaMemcpyDefault, h->stream));
  if (int rc = issue(apply_update != 0, weights ? h->weights : nullptr)) return rc;
  if (apply_update) ++h->n_updates;
  if (td_out) CK(cudaMemcpyAsync(td_out, h->td, B * A * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  return 0;
}

// ------------------------------------------------------------------------------------------------------------- observe path
namespace {
// the refusals every observe call makes
int ql_observe_checks(const QLearner* h, int n, int update_stats) {
  if (n < 1 || n > h->stage_rows)
    return b2g_fail(B2G_EINVAL, "observe: n must be in [1, " + std::to_string(h->stage_rows) + "] (the staging holds max(batch, 256) frames)");
  if (update_stats && !h->rms.on())
    return b2g_fail(B2G_ESTATE, std::string("update_stats needs device statistics: call ") + h->rms.set_call + " first");
  return 0;
}

// the staging buffers, on first use
int ql_observe_alloc(QLearner* h) {
  if (h->ob_rows[0]) return 0;
  const size_t R = h->stage_rows, E = h->E;
  for (int k = 0; k < 2; ++k)
    if (int rc = dev_alloc(h->allocs, h->stream, &h->ob_rows[k], (R + h->B) * E)) return rc;
  if (int rc = dev_alloc(h->allocs, h->stream, &h->ob_reset, R * E)) return rc;
  if (int rc = dev_alloc(h->allocs, h->stream, &h->ob_act, R * h->A)) return rc;
  if (int rc = dev_alloc(h->allocs, h->stream, &h->ob_rew, R)) return rc;
  if (int rc = dev_alloc(h->allocs, h->stream, &h->ob_done, R)) return rc;
  return dev_alloc(h->allocs, h->stream, &h->ob_idx, R * h->A);
}
}  // namespace

int ql_observe_act(QLearner* h, const float* obs, int n, int update_stats, bool acting, const std::function<int(const float*)>& act) {
  if (int rc = ql_observe_checks(h, n, obs ? update_stats : 0)) return rc;
  if (!obs && h->ob_n == 0) return b2g_fail(B2G_ESTATE, "observe_act: no staged observations (pass obs first)");
  if (!obs && n != h->ob_n) return b2g_fail(B2G_EINVAL, "observe_act: n differs from the number of staged observations");
  CK(cudaSetDevice(h->device));
  if (int rc = ql_observe_alloc(h)) return rc;
  float* cur = h->ob_rows[h->ob_k];
  if (obs) {
    if (int rc = h->rms.stage_frames(cur, obs, n, h->stream)) return rc;
    if (update_stats) h->rms.merge(cur, nullptr, nullptr, n, h->stream);
    h->ob_n = n;
    h->ob_fid.assign((size_t)n, -1);
  }
  if (acting)
    if (int rc = act(cur)) return rc;
  CK(cudaStreamSynchronize(h->stream));     // caller-owned arrays are copied, the actions are the result of the call
  CK(cudaGetLastError());
  return 0;
}

int ql_observe_add(QLearner* h, const float* act, const float* rew, const float* next_obs, const float* done, const float* reset_obs,
                   int n, int update_stats, const std::function<int()>& check) {
  if (int rc = ql_observe_checks(h, n, update_stats)) return rc;
  if (h->ob_n == 0)
    return b2g_fail(B2G_ESTATE, std::string("observe_add: no staged observations (call b2g_") + h->abi + "_observe_act first)");
  if (n != h->ob_n) return b2g_fail(B2G_EINVAL, "observe_add: n differs from the number of staged observations");
  if (n > h->buffer_capacity) return b2g_fail(B2G_EINVAL, "observe_add: n exceeds buffer_capacity");
  if (h->replay.ring.dedup && 2 * (int64_t)n > h->replay.ring.frame_cap)
    return b2g_fail(B2G_EINVAL, "observe_add: 2 n rows exceed frame_capacity (replay_frames)");
  int n_done = 0;
  for (int i = 0; i < n; ++i) n_done += done[i] != 0.f;
  if (n_done && !reset_obs) return b2g_fail(B2G_EINVAL, "observe_add: an env finished but reset_obs is NULL");
  if (check)
    if (int rc = check()) return rc;
  CK(cudaSetDevice(h->device));
  if (int rc = ql_observe_alloc(h)) return rc;
  const size_t E = h->E, A = h->A, fb = E * sizeof(float);
  float* cur = h->ob_rows[h->ob_k];
  float* nxt = h->ob_rows[h->ob_k ^ 1];
  if (int rc = h->rms.stage_frames(nxt, next_obs, n, h->stream)) return rc;
  if (int rc = h->rms.upload(h->ob_act, act, n * A * sizeof(float), h->stream)) return rc;
  if (int rc = h->rms.upload(h->ob_rew, rew, n * sizeof(float), h->stream)) return rc;
  if (int rc = h->rms.upload(h->ob_done, done, n * sizeof(float), h->stream)) return rc;
  if (n_done)
    if (int rc = h->rms.stage_reset_frames(h->ob_reset, reset_obs, done, h->ob_done, n, n_done, h->stream)) return rc;
  // the transitions: obs = the staged rows, next_obs = the uploaded rows (what the caller passes as a finished env's next_obs)
  TransitionReplay& rp = h->replay;
  if (rp.framed()) {
    // env i's staged row is the frame its previous transition's next_obs took, unless the env was reset since: shared without
    // comparing; a reset frame (ob_fid -1) takes a frame of its own here, when it is first used as obs
    std::vector<int64_t> next_ids((size_t)n);
    if (int rc = rp.add_linked(cur, nxt, h->ob_fid.data(), h->ob_act, h->ob_rew, h->ob_done, n, next_ids.data(), h->counters, h->stream))
      return rc;
    for (int i = 0; i < n; ++i) h->ob_fid[i] = done[i] != 0.f ? -1 : next_ids[i];
  } else {
    const int64_t new_size = std::min<int64_t>(rp.cap, rp.size + n);
    ql_commit_kernel<<<n, 256, 0, h->stream>>>(cur, nxt, h->ob_act, h->ob_rew, h->ob_done, (int)E, (int)A, rp.pos, rp.cap, rp.obs, rp.next,
                                               rp.act, rp.rew, rp.done, h->counters, new_size);
    rp.insert_max_prio(rp.pos, n, h->stream);     // as in replay_add
  }
  // VecNormalize's step_wait merges the frames the VecEnv returned: a finished env's reset frame, not its terminal observation
  if (update_stats) h->rms.merge(nxt, n_done ? h->ob_reset : nullptr, h->ob_done, n, h->stream);
  // the new rows become the current observations; a finished env continues from the frame its reset returned
  for (int i = 0; i < n; ++i)
    if (done[i] != 0.f) CK(cudaMemcpyAsync(nxt + i * E, h->ob_reset + i * E, fb, cudaMemcpyDeviceToDevice, h->stream));
  if (!rp.framed()) rp.advance(n);
  h->ob_k ^= 1;
  CK(cudaStreamSynchronize(h->stream));     // host arrays are caller-owned: copied before return
  CK(cudaGetLastError());
  return 0;
}

int ql_set_obs_encoder(QLearner* h, const b2g_encoder* enc, int tail) {
  if (enc)
    if (int rc = obs_rms_check_encoder(h, enc, tail)) return rc;
  return obs_rms_attach_encoder(h, enc, tail);
}

// ------------------------------------------------------------------------------------------------------------- training state
namespace {
// sections 2.. (parameters .. prioritised-replay scalars, then obs_rms when the handle owns it) of a handle holding `live`
// replay rows
std::vector<StateSection> ql_device_sections(QLearner* h, ObsRms* rms, int64_t live, int64_t lo = 0, int64_t hi = 0) {
  std::vector<StateSection> s = adam_sections(h->P, 2 * h->n_train, h->Mo, h->Vo, h->n_train);
  for (auto& r : h->replay.state_sections(live, lo, hi)) s.push_back(std::move(r));
  for (auto& r : h->replay.per_sections()) s.push_back(std::move(r));
  if (rms && rms->on()) s.push_back(rms_section(&rms->count, rms->mean, rms->var, h->E));
  return s;
}
}  // namespace

int ql_state_save(QLearner* h, const char* path, uint32_t kind, const std::vector<FpField>& fp, ObsRms* rms, const char* refusal) {
  if (!h || !path) return b2g_fail(B2G_EINVAL, "NULL argument");
  B2G_USABLE(h);
  if (refusal) return b2g_fail(B2G_ESTATE, refusal);
  CK(cudaSetDevice(h->device));
  CK(cudaStreamSynchronize(h->stream));
  long long cnt[8];
  CK(cudaMemcpy(cnt, h->counters, sizeof cnt, cudaMemcpyDeviceToHost));
  uint32_t eps_bits;
  memcpy(&eps_bits, &h->eps_value, sizeof eps_bits);
  std::vector<int64_t> hv = h->replay.state_host(h->n_updates, (int64_t)eps_bits);
  const FrameRing& ring = h->replay.ring;
  std::vector<StateSection> secs = host_sections(hv.data(), hv.size() * sizeof(int64_t), cnt, sizeof cnt);
  for (auto& s : ql_device_sections(h, rms, h->replay.size, ring.frame_lo(), ring.next_fid)) secs.push_back(std::move(s));
  return state_write(path, kind, fp_with_rms(fp_with_frames(fp, ring.frame_cap), rms && rms->on()), secs);
}

int ql_state_load(QLearner* h, const char* path, uint32_t kind, const std::vector<FpField>& fp, ObsRms* rms, const char* refusal,
                  const char* learner, const std::function<void()>& restore) {
  if (!h || !path) return b2g_fail(B2G_EINVAL, "NULL argument");
  if (refusal) return b2g_fail(B2G_ESTATE, refusal);
  CK(cudaSetDevice(h->device));
  // ---- everything is checked before the handle changes
  StateReader rd;
  TransitionReplay& rp = h->replay;
  if (int rc = state_open_replay(rd, path, kind, fp, rp.ring.frame_cap, rms && rms->on(), rms ? rms->set_call : "")) return rc;
  if (int rc = state_check_tags(rd, ql_device_sections(h, rms, 0), learner)) return rc;
  long long cnt[8];
  if (rd.bytes(1) != sizeof cnt) return b2g_fail(B2G_EINVAL, "training-state section lengths do not match this handle's configuration");
  std::vector<int64_t> hv;
  FrameRing ring;
  if (int rc = rp.state_host_read(rd, &hv, &ring)) return rc;
  const std::vector<StateSection> dev = ql_device_sections(h, rms, hv[0], ring.frame_lo(), ring.next_fid);
  if (int rc = state_check_lengths(rd, dev)) return rc;
  if (int rc = rd.read_host(1, cnt, sizeof cnt)) return rc;
  // ---- from here on a failure leaves the handle unusable until a load succeeds
  CK(cudaStreamSynchronize(h->stream));
  return state_read_device(rd, dev, &h->broken, [&] {
    if (rms && rms->on()) {
      rms->derive(h->stream);
      CK(cudaStreamSynchronize(h->stream));
    }
    if (restore) restore();
    CK(cudaMemcpy(h->counters, cnt, sizeof cnt, cudaMemcpyHostToDevice));
    rp.ring = ring;
    rp.size = hv[0]; rp.pos = hv[1]; h->n_updates = hv[2];
    const uint32_t eps_bits = (uint32_t)hv[3];
    memcpy(&h->eps_value, &eps_bits, sizeof eps_bits);
    // the captured step graph stays valid: it holds device pointers and configuration; size and Philox step are device counters
    return mlog_rebase(&h->mlog, h->counters + 3, h->stream);     // the restored counter: rows before it are not pending
  });
}

int ql_metrics_log(QLearner* h, int capacity, int cols) {
  B2G_USABLE(h);
  if (!h || capacity < 0) return b2g_fail(B2G_EINVAL, "bad argument");
  CK(cudaSetDevice(h->device));
  if (int rc = mlog_enable(&h->mlog, capacity, cols, h->counters + 3, h->stream)) return rc;
  // the step gains or loses its append node: capture again at the next step
  if (h->graph_exec) { cudaGraphExecDestroy(h->graph_exec); h->graph_exec = nullptr; }
  return 0;
}

int ql_metrics_drain(QLearner* h, float* rows, int max_rows, int64_t* first_step, int* n_rows, int64_t* lost,
                     const std::function<void(float*)>& fix) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  CK(cudaSetDevice(h->device));
  return mlog_drain(&h->mlog, h->counters + 3, h->stream, rows, max_rows, first_step, n_rows, lost, fix);
}

}  // namespace b2g
