// The observation encoder of a learner handle (b2g_sac_set_obs_encoder / b2g_bdq_set_obs_encoder; encoder.cu): a frozen copy
// of an encoder handle's geometry and weights on the learner's device, run on the learner's stream over the raw rows that
// b2g_*_observe_* upload.  A raw row is [H*W*C pixels (HWC) | tail floats]; the encoded row it becomes is
// [encoding_dim | tail], at the learner's row stride E = encoding_dim + tail.
#pragma once
#include <cuda_runtime.h>

#include "../../include/b200grasp.h"

namespace b2g {

struct EncStage;

// Checks, before any CUDA call, what only the encoder knows (B2G_EINVAL: encoding_dim + tail != obs_dim, tail < 0, another
// device; B2G_ESTATE: a layer without weights), then builds the stage for batches up to `rows` on the current device.
int enc_stage_check(const b2g_encoder* enc, int device, int tail, int obs_dim);
int enc_stage_create(const b2g_encoder* enc, int rows, int tail, cudaStream_t s, EncStage** out);
// Frees the stage's device memory (the caller has drained the stream it ran on).
void enc_stage_destroy(EncStage* st);
// Floats per raw row (H*W*C + tail).
int enc_stage_row_floats(const EncStage* st);
// Upload buffer `which` (0 = every env's frame, 1 = reset frames of finished envs), [rows][row_floats].
float* enc_stage_raw(EncStage* st, int which);
// Encodes raw rows of buffer `which` into dst ([.][E], E = encoding_dim + tail), enqueued on s.  which == 0: rows 0 .. n-1.
// which == 1: only the rows i < n with done[i] != 0 (device flags), n_done of them; the other rows of buffer 1 and of dst are
// not touched.
int enc_stage_encode(EncStage* st, int which, const float* done, int n, int n_done, float* dst, cudaStream_t s);

}  // namespace b2g
