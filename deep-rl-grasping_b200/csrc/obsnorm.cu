// VecNormalize's observation statistics on the device, and the actor side of the learn loop fed from one upload per frame
// (b2g_sac_observe_act / b2g_sac_observe_add / b2g_obs_rms_set / b2g_obs_rms_get; contracts in include/b200grasp.h).  The
// statistics, their staging and their entry-point bodies are ObsRms (obsnorm.cuh), which the BDQ learner's b2g_bdq_observe_*
// (bdq.cu) use too, over the flat layout.
//
// obs_rms = (mean[E], var[E], count) in float64 over the caller's observation layout, the object [SB2]
// common/running_mean_std.py keeps on the host.  obs_rms_update_kernel merges the n frames of one call into it with the
// parallel-moments rule of RunningMeanStd.update_from_moments and rewrites, in the same pass, the entries of d_mean / d_istd
// (compact-row layout) that the gather of the gradient step and of policy inference read.  Everything is enqueued on the
// handle's stream, so a step sampled after a call normalises with the statistics that call left.
//
// Which frames are merged, and when, is [SB2] VecNormalize's rule: reset() merges the reset frames (b2g_sac_observe_act with
// obs != NULL), step_wait() merges the n frames the VecEnv returned, which for a finished env is the frame its auto-reset
// returned and NOT the terminal observation (b2g_sac_observe_add: next_obs_i, or reset_obs_i where done_i).  The terminal
// observation goes into the replay only.
//
// Every copy and kernel of a call is enqueued on the handle's stream and the call synchronises it once before it returns, as
// b2g_replay_add and b2g_sac_act do: the caller's arrays are free on return.
//
// With an observation encoder (b2g_sac_set_obs_encoder) the frames uploaded are raw depth rows; the encoder stage (encoder.cu)
// turns them into the encoded rows of ob_full on the device, and everything after it runs on those unchanged.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "obsnorm.cuh"
#include "sac_internal.cuh"

namespace b2g {
namespace {

// element e of frame i: a + i E, or (RESET) the reset frame b + i E where env i finished (done[i] != 0)
template <bool RESET>
__device__ __forceinline__ float frame_value(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ done,
                                             int i, int E, int e) {
  const float* f = a;
  if (RESET) f = done[i] != 0.f ? b : a;
  return f[(size_t)i * E + e];
}

// One thread per element e of the caller's layout.  The n
// values are summed in frame order 0 .. n-1 (mean, then squared deviations from it), so the result does not depend on the
// grid; consecutive threads read consecutive floats of every frame.  n == 0 only derives the table.
// Cfull > 0: [HW][Cfull] observations whose compact row keeps the image planes and pixel [0,0] of the last plane (index npx).
// Cfull == 0: the flat layout, table entry e = element e (SAC's MLP rows, BDQ's [obs_dim] rows).
template <bool RESET>
__global__ void __launch_bounds__(256) obs_rms_update_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                              const float* __restrict__ done, int n, int E, double count, double eps,
                                                              double* __restrict__ mean, double* __restrict__ var,
                                                              double* __restrict__ d_mean, double* __restrict__ d_istd, int Cfull, int npx) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  double m = mean[e], v = var[e];
  if (n > 0) {
    double s = 0.0;
    for (int i = 0; i < n; ++i) s += (double)frame_value<RESET>(a, b, done, i, E, e);
    const double bm = s / n;
    double q = 0.0;
    for (int i = 0; i < n; ++i) {
      const double d = (double)frame_value<RESET>(a, b, done, i, E, e) - bm;
      q += d * d;
    }
    const double bv = q / n, delta = bm - m, tot = count + n;
    m = m + delta * n / tot;
    v = (v * count + bv * n + delta * delta * count * n / tot) / tot;
    mean[e] = m;
    var[e] = v;
  }
  int r = e;
  if (Cfull > 0) {
    const int pix = e / Cfull, c = e - pix * Cfull;
    r = c < Cfull - 1 ? pix * (Cfull - 1) + c : (pix == 0 ? npx : -1);
  }
  if (r >= 0) {
    d_mean[r] = m;
    d_istd[r] = 1.0 / sqrt(v + eps);
  }
}

int ensure_staging(b2g_sac* h) {
  if (h->ob_act) return 0;
  const size_t R = h->stage_rows;
  for (int k = 0; k < 2; ++k) {
    if (int rc = dev_alloc(h->allocs, h->stream, &h->ob_full[k], R * h->E)) return rc;
    if (int rc = dev_alloc(h->allocs, h->stream, &h->ob_rows[k], (R + h->B) * h->Ec)) return rc;
  }
  if (int rc = dev_alloc(h->allocs, h->stream, &h->ob_act, R * h->A)) return rc;
  if (int rc = dev_alloc(h->allocs, h->stream, &h->ob_rew, R)) return rc;
  return dev_alloc(h->allocs, h->stream, &h->ob_done, R);
}

// every value of an 8-bit plane is an integer in [0, 255] (what b2g_replay_add refuses on the device, checked here on the
// host so that nothing is enqueued for a refused call)
bool u8_values_ok(const b2g_sac* h, const float* frame) {
  const int Cfull = h->Cobs, HW = h->Hi * h->Wi;
  for (int c = 0; c < h->Cimg; ++c) {
    if (!(h->u8_mask >> c & 1)) continue;
    for (int p = 0; p < HW; ++p) {
      const float v = frame[(size_t)p * Cfull + c];
      if (!(v >= 0.f && v <= 255.f && v == rintf(v) && !signbit(v))) return false;
    }
  }
  return true;
}

int check_frames(const b2g_sac* h, const float* frames, const float* only_where, int n) {
  if (!h->u8_mask) return 0;
  for (int i = 0; i < n; ++i)
    if ((!only_where || only_where[i] != 0.f) && !u8_values_ok(h, frames + (size_t)i * h->E))
      return b2g_fail(B2G_EINVAL, "observe: a value of an 8-bit plane is not an integer in [0, 255]");
  return 0;
}

// caller-layout frames [n][E] -> compact rows [n][Ec]
int to_rows(b2g_sac* h, const float* full, float* rows, int row0, int n) {
  if (h->cnn) compact_rows(full, rows, row0, (long long)h->stage_rows + h->B, n, h->Hi * h->Wi, h->Cimg, h->Cobs, h->stream);
  else CK(cudaMemcpyAsync(rows + (size_t)row0 * h->Ec, full, (size_t)n * h->E * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
  return 0;
}

int common_checks(b2g_sac* h, int n, int update_stats) {
  if (h->pipe_pending) return b2g_fail(B2G_ESTATE, "a host-pipelined step is in flight: call b2g_sac_pipeline_flush first");
  if (n < 1 || n > h->stage_rows)
    return b2g_fail(B2G_EINVAL, "observe: n must be in [1, " + std::to_string(h->stage_rows) + "] (the staging holds max(batch, 256) frames)");
  if (update_stats && !h->rms.on())
    return b2g_fail(B2G_ESTATE, "update_stats needs device statistics: call b2g_obs_rms_set first");
  return 0;
}

}  // namespace

void obs_rms_update_launch(const float* a, const float* b, const float* done, int n, int E, double count, double eps, double* mean,
                           double* var, double* d_mean, double* d_istd, int Cfull, int npx, cudaStream_t s) {
  const dim3 grid((E + 255) / 256);
  if (b) obs_rms_update_kernel<true><<<grid, 256, 0, s>>>(a, b, done, n, E, count, eps, mean, var, d_mean, d_istd, Cfull, npx);
  else obs_rms_update_kernel<false><<<grid, 256, 0, s>>>(a, b, done, n, E, count, eps, mean, var, d_mean, d_istd, Cfull, npx);
}

void ObsRms::merge(const float* a, const float* b, const float* done, int n, cudaStream_t s) {
  obs_rms_update_launch(a, b, done, n, E, count, eps, mean, var, d_mean, d_istd, Cfull, npx, s);
  count += n;
}

int ObsRms::set(const double* m, const double* v, double c, int device, int nranks, std::vector<void*>& allocs, cudaStream_t s) {
  if (!(c >= 0.0) || !std::isfinite(c)) return b2g_fail(B2G_EINVAL, "obs_rms_set: count must be finite and >= 0");
  for (int e = 0; e < E; ++e)
    if (!std::isfinite(m[e]) || !(v[e] >= 0.0) || !std::isfinite(v[e]))
      return b2g_fail(B2G_EINVAL, "obs_rms_set: mean must be finite and var finite and >= 0 (element " + std::to_string(e) + ")");
  if (nranks > 1)
    return b2g_fail(B2G_ESTATE, "device observation statistics are per handle: with nranks > 1 every rank would own different ones");
  CK(cudaSetDevice(device));
  if (!mean) {     // one allocation for both arrays: it either exists or it does not
    double* mv = nullptr;
    if (int rc = dev_alloc(allocs, s, &mv, 2 * (size_t)E, false)) return rc;
    mean = mv;
    var = mv + E;
  }
  CK(cudaMemcpyAsync(mean, m, E * sizeof(double), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(var, v, E * sizeof(double), cudaMemcpyHostToDevice, s));
  up_observe += (int64_t)(2 * E * sizeof(double));
  count = c;
  derive(s);
  CK(cudaStreamSynchronize(s));     // host arrays are caller-owned: copied before return
  return 0;
}

int ObsRms::norm_stats(const double* m, const double* v, double eps_, int device, int nranks, std::vector<void*>& allocs, cudaStream_t s) {
  const bool eps_changed = eps_ != eps;
  eps = eps_;
  if (!on()) return 0;
  if (m && v) return set(m, v, count, device, nranks, allocs, s);
  if (eps_changed) derive(s);
  return 0;
}

int ObsRms::upload(void* dst, const void* src, size_t bytes, cudaStream_t s) {
  CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s));
  up_observe += (int64_t)bytes;
  return 0;
}

int ObsRms::stage_frames(float* dst, const float* obs, int n, cudaStream_t s) {
  if (!enc) return upload(dst, obs, (size_t)n * E * sizeof(float), s);
  if (int rc = upload(enc_stage_raw(enc, 0), obs, (size_t)n * enc_stage_row_floats(enc) * sizeof(float), s)) return rc;
  return enc_stage_encode(enc, 0, nullptr, n, 0, dst, s);
}

int ObsRms::stage_reset_frames(float* dst, const float* reset_obs, const float* done, const float* d_done, int n, int n_done,
                               cudaStream_t s) {
  const size_t rw = enc ? enc_stage_row_floats(enc) : E;
  float* up = enc ? enc_stage_raw(enc, 1) : dst;
  for (int i = 0; i < n; ++i)
    if (done[i] != 0.f)
      if (int rc = upload(up + i * rw, reset_obs + i * rw, rw * sizeof(float), s)) return rc;
  return enc ? enc_stage_encode(enc, 1, d_done, n, n_done, dst, s) : 0;
}

}  // namespace b2g

extern "C" {

int b2g_obs_rms_set(b2g_sac* h, const double* mean, const double* var, double count) { return obs_rms_set(h, mean, var, count); }
int b2g_obs_rms_get(b2g_sac* h, double* mean, double* var, double* count) { return obs_rms_get(h, mean, var, count); }
int b2g_upload_bytes(const b2g_sac* h, int64_t* observe_bytes, int64_t* other_bytes) {
  return obs_rms_upload_bytes(h, observe_bytes, other_bytes);
}

int b2g_sac_set_obs_encoder(b2g_sac* h, const b2g_encoder* enc, int tail) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  if (enc) {
    if (h->cnn) return b2g_fail(B2G_EINVAL, "set_obs_encoder: the CNN policy reads images itself; an encoder feeds the MLP policy");
    if (int rc = obs_rms_check_encoder(h, enc, tail)) return rc;
  }
  if (h->pipe_pending) return b2g_fail(B2G_ESTATE, "a host-pipelined step is in flight: call b2g_sac_pipeline_flush first");
  if (int rc = obs_rms_attach_encoder(h, enc, tail)) return rc;
  h->ob_fid.clear();
  return 0;
}

int b2g_sac_observe_act(b2g_sac* h, const float* obs, int n, int update_stats, int deterministic, float* act_out) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  if (!obs && !act_out) return b2g_fail(B2G_EINVAL, "observe_act: nothing to do (obs and act_out are NULL)");
  if (int rc = common_checks(h, n, obs ? update_stats : 0)) return rc;
  if (!obs && h->ob_n == 0) return b2g_fail(B2G_ESTATE, "observe_act: no staged observations (pass obs first)");
  if (!obs && n != h->ob_n) return b2g_fail(B2G_EINVAL, "observe_act: n differs from the number of staged observations");
  if (obs)
    if (int rc = check_frames(h, obs, nullptr, n)) return rc;
  CK(cudaSetDevice(h->cfg.device));
  if (int rc = ensure_staging(h)) return rc;
  if (obs) {
    if (int rc = h->rms.stage_frames(h->ob_full[0], obs, n, h->stream)) return rc;
    if (update_stats) h->rms.merge(h->ob_full[0], nullptr, nullptr, n, h->stream);
    if (int rc = to_rows(h, h->ob_full[0], h->ob_rows[h->ob_k], 0, n)) return rc;
    h->ob_fid.assign((size_t)n, -1);
    h->ob_n = n;
    if (!act_out) CK(cudaStreamSynchronize(h->stream));     // host arrays are caller-owned: copied before return
  }
  if (act_out) {
    const size_t A = h->A;
    for (int k = 0; k < n; k += h->B) {
      const int chunk = std::min(h->B, n - k);
      if (int rc = sac_act_rows(h, h->ob_rows[h->ob_k] + (size_t)k * h->Ec, chunk, deterministic)) return rc;
      CK(cudaMemcpyAsync(act_out + (size_t)k * A, h->pi_out, chunk * A * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));      // the actions are the result of the call
    }
  }
  CK(cudaGetLastError());
  return 0;
}

int b2g_sac_observe_add(b2g_sac* h, const float* act, const float* rew, const float* next_obs, const float* done,
                        const float* reset_obs, int n, int update_stats) {
  B2G_USABLE(h);
  if (!h || !act || !rew || !next_obs || !done) return b2g_fail(B2G_EINVAL, "NULL argument");
  if (int rc = common_checks(h, n, update_stats)) return rc;
  if (h->ob_n == 0) return b2g_fail(B2G_ESTATE, "observe_add: no staged observations (call b2g_sac_observe_act first)");
  if (n != h->ob_n) return b2g_fail(B2G_EINVAL, "observe_add: n differs from the number of staged observations");
  if (h->replay.ring.dedup && 2 * (int64_t)n > h->replay.ring.frame_cap)
    return b2g_fail(B2G_EINVAL, "observe_add: 2 n rows exceed frame_capacity");
  int n_done = 0;
  for (int i = 0; i < n; ++i) n_done += done[i] != 0.f;
  if (n_done && !reset_obs) return b2g_fail(B2G_EINVAL, "observe_add: an env finished but reset_obs is NULL");
  if (int rc = check_frames(h, next_obs, nullptr, n)) return rc;
  if (n_done)
    if (int rc = check_frames(h, reset_obs, done, n)) return rc;
  CK(cudaSetDevice(h->cfg.device));
  const size_t E = h->E, A = h->A;
  if (int rc = h->rms.stage_frames(h->ob_full[0], next_obs, n, h->stream)) return rc;
  if (int rc = h->rms.upload(h->ob_act, act, n * A * sizeof(float), h->stream)) return rc;
  if (int rc = h->rms.upload(h->ob_rew, rew, n * sizeof(float), h->stream)) return rc;
  if (int rc = h->rms.upload(h->ob_done, done, n * sizeof(float), h->stream)) return rc;
  if (n_done)
    if (int rc = h->rms.stage_reset_frames(h->ob_full[1], reset_obs, done, h->ob_done, n, n_done, h->stream)) return rc;
  // the transitions: obs = the staged rows (linked to their replay frame where one holds them), next_obs = the new rows
  float* cur = h->ob_rows[h->ob_k];
  float* nxt = h->ob_rows[h->ob_k ^ 1];
  if (int rc = to_rows(h, h->ob_full[0], nxt, 0, n)) return rc;
  std::vector<int64_t> next_fid((size_t)n);
  if (int rc = h->replay.add_linked(cur, nxt, h->ob_fid.data(), h->ob_act, h->ob_rew, h->ob_done, n, next_fid.data(), h->counters,
                                    h->stream))
    return rc;
  if (update_stats) h->rms.merge(h->ob_full[0], n_done ? h->ob_full[1] : nullptr, h->ob_done, n, h->stream);
  // the new rows become the current observations; a finished env continues from the frame its reset returned
  for (int i = 0; i < n; ++i) {
    h->ob_fid[i] = next_fid[i];
    if (done[i] != 0.f) {
      if (int rc = to_rows(h, h->ob_full[1] + i * E, nxt, i, 1)) return rc;
      h->ob_fid[i] = -1;
    }
  }
  h->ob_k ^= 1;
  CK(cudaStreamSynchronize(h->stream));     // host arrays are caller-owned: copied before return
  CK(cudaGetLastError());
  return 0;
}

}  // extern "C"
