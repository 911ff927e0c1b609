// VecNormalize's observation statistics on the device (obs_rms) and the frame staging of the observe path, one implementation
// for the SAC (obsnorm.cu), BDQ / DQN (q_learner.cu) and PPO2 / TRPO (actor_critic.cu) handles.  A handle owns one ObsRms as its
// member `rms`; the templates below are the bodies of its b2g_*obs_rms_set / _get and b2g_*upload_bytes, and the checks and
// attach of b2g_*_set_obs_encoder.  They read the handle's cfg.device, cfg.nranks, allocs, stream, stage_rows and ob_n.
#pragma once
#include <cuda_runtime.h>

#include <cmath>
#include <string>
#include <vector>

#include "enc_stage.cuh"
#include "host.cuh"

namespace b2g {

struct ObsRms {
  // float64 mean / var [E] over the caller's observation layout, one allocation (created by the set call); the count stays on
  // the host: count + n is the same float64 sum there
  double *mean = nullptr, *var = nullptr;
  double count = 0.0;
  double eps = 1e-8;                  // VecNormalize.epsilon of the last set_norm_stats
  int64_t up_observe = 0, up_other = 0;   // host->device bytes: observe_* / obs_rms_set, and act + replay_add + set_norm_stats
  EncStage* enc = nullptr;            // set_obs_encoder: observe_* take raw rows and encode them into the staged rows
  int E = 0;                          // caller-layout width
  int Cfull = 0, npx = 0;             // the table layout (obs_rms_update_launch)
  double *d_mean = nullptr, *d_istd = nullptr;   // the table the gather reads
  const char* set_call = "";          // the entry point that creates obs_rms, named in error text
  bool on() const { return mean != nullptr; }

  // obs_rms_set's body (the caller has checked its handle and pointers): the values checked, obs_rms created on first use, the
  // arrays uploaded and the table derived; synchronises s
  int set(const double* m, const double* v, double c, int device, int nranks, std::vector<void*>& allocs, cudaStream_t s);
  // The obs_rms branch of set_norm_stats: records eps and, when obs_rms exists, lets statistics passed here replace it (count
  // kept) or derives the table again when only eps changed.  The caller uploads no statistics of its own while on().
  int norm_stats(const double* m, const double* v, double eps_, int device, int nranks, std::vector<void*>& allocs, cudaStream_t s);

  // merges the n frames a[i] (b[i] where done[i] != 0 when b != nullptr) and rewrites the table, enqueued on s
  void merge(const float* a, const float* b, const float* done, int n, cudaStream_t s);
  // rewrites the table from obs_rms and eps, enqueued on s
  void derive(cudaStream_t s) { merge(nullptr, nullptr, nullptr, 0, s); }
  // a counted observe-path upload
  int upload(void* dst, const void* src, size_t bytes, cudaStream_t s);
  // the n frames of a call -> rows [n][E] at dst: uploaded as they are or, with an observation encoder, as raw rows it encodes
  // there
  int stage_frames(float* dst, const float* obs, int n, cudaStream_t s);
  // the reset frames of the n_done finished envs -> row i of dst; only those cross the bus and, with an observation encoder,
  // only those are encoded (it reads the device flags d_done, uploaded before)
  int stage_reset_frames(float* dst, const float* reset_obs, const float* done, const float* d_done, int n, int n_done, cudaStream_t s);
};

template <class H>
int obs_rms_set(H* h, const double* mean, const double* var, double count) {
  B2G_USABLE(h);
  if (!h || !mean || !var) return b2g_fail(B2G_EINVAL, "NULL argument");
  return h->rms.set(mean, var, count, h->cfg.device, h->cfg.nranks, h->allocs, h->stream);
}

template <class H>
int obs_rms_get(H* h, double* mean, double* var, double* count) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  const ObsRms& r = h->rms;
  if (!r.mean) return b2g_fail(B2G_ESTATE, std::string("the handle has no device statistics: call ") + r.set_call + " first");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  if (mean) CK(cudaMemcpy(mean, r.mean, r.E * sizeof(double), cudaMemcpyDeviceToHost));
  if (var) CK(cudaMemcpy(var, r.var, r.E * sizeof(double), cudaMemcpyDeviceToHost));
  if (count) *count = r.count;
  return 0;
}

template <class H>
int obs_rms_upload_bytes(const H* h, int64_t* observe_bytes, int64_t* other_bytes) {
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  if (observe_bytes) *observe_bytes = h->rms.up_observe;
  if (other_bytes) *other_bytes = h->rms.up_other;
  return 0;
}

// set_obs_encoder's refusals of an encoder (enc != null): what the encoder checks, and a data-parallel handle
template <class H>
int obs_rms_check_encoder(const H* h, const b2g_encoder* enc, int tail) {
  if (int rc = enc_stage_check(enc, h->cfg.device, tail, h->rms.E)) return rc;
  if (h->cfg.nranks > 1)
    return b2g_fail(B2G_ESTATE, "set_obs_encoder: the observe path is per handle: with nranks > 1 every rank would encode its own");
  return 0;
}

// set_obs_encoder once every refusal passed: a stage of stage_rows rows (none when enc is null) replaces the old one; the
// staged observations were in the other layout.
template <class H>
int obs_rms_attach_encoder(H* h, const b2g_encoder* enc, int tail) {
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  EncStage* st = nullptr;
  if (enc)
    if (int rc = enc_stage_create(enc, h->stage_rows, tail, h->stream, &st)) return rc;
  enc_stage_destroy(h->rms.enc);
  h->rms.enc = st;
  h->ob_n = 0;
  return 0;
}

}  // namespace b2g
