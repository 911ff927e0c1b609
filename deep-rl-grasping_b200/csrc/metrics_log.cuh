// Per-step metrics ring of the replay learners (SAC, BDQ, DQN): every applied gradient step appends its K loss scalars to a
// device ring [cap][K] at row (n_updates - 1) % cap, where n_updates is the handle's device optimiser-step counter
// (counters[3], advanced by prep_kernel).  The append is one tiny kernel at the end of the step, so it is captured into the
// step graph and works across graph replays and n_steps > 1 calls without a host round trip.  The host drains the rows
// written since the last drain in batches (b2g_*_metrics_drain).  A handle whose log is off adds no node.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <functional>

namespace b2g {

constexpr int MLOG_MAX_K = 8;

// the device scalars one row copies, in column order
struct MetricsLogSrc {
  const float* src[MLOG_MAX_K];
  int K;
};

struct MetricsLog {
  int cap = 0, K = 0;
  float* ring = nullptr;         // device [cap][K]
  float* h_rows = nullptr;       // pinned [cap][K]: drain staging
  long long* h_step = nullptr;   // pinned: the step counter read by a drain
  long long drained = 0;         // counter value up to which rows were handed out or counted lost
  bool on() const { return cap > 0; }
};

// cap > 0: (re)allocates a ring of cap rows of K floats and starts it at the current counter value (nothing pending);
// cap == 0: frees it.  Synchronises `s`.
int mlog_enable(MetricsLog* m, int cap, int K, const long long* d_step, cudaStream_t s);
void mlog_free(MetricsLog* m);
// enqueues the append of one row on `s` (behind the step's optimiser launch)
void mlog_append(const MetricsLog& m, const MetricsLogSrc& src, const long long* d_step, cudaStream_t s);
// after the counter was overwritten (training-state load): nothing pending.  Synchronises `s`.
int mlog_rebase(MetricsLog* m, const long long* d_step, cudaStream_t s);
// Synchronises `s`, then copies up to max_rows of the rows written since the last drain (oldest first) to rows[n][K], each
// passed through fix (the handle's host-side finishing: 1/nranks, sqrt, exp).  *first_step = n_updates of the first row;
// *lost = rows overwritten before they were drained (they are skipped).  Rows beyond max_rows stay for the next drain.
int mlog_drain(MetricsLog* m, const long long* d_step, cudaStream_t s, float* rows, int max_rows, int64_t* first_step,
               int* n_rows, int64_t* lost, const std::function<void(float*)>& fix);

}  // namespace b2g
