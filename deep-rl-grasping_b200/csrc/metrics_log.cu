// Per-step metrics ring of the replay learners (metrics_log.cuh).
#include <string.h>

#include <algorithm>

#include "host.cuh"
#include "metrics_log.cuh"

namespace b2g {
namespace {

// one thread per column; step[0] already counts the step that wrote the scalars (prep_kernel advanced it)
__global__ void metrics_log_append_kernel(float* __restrict__ ring, int cap, int K, const long long* __restrict__ step,
                                          MetricsLogSrc src) {
  const int k = threadIdx.x;
  if (k >= K) return;
  const long long t = step[0] - 1;
  ring[(size_t)(t % cap) * K + k] = *src.src[k];
}

int read_step(MetricsLog* m, const long long* d_step, cudaStream_t s, long long* out) {
  CK(cudaMemcpyAsync(m->h_step, d_step, sizeof(long long), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  *out = *m->h_step;
  return 0;
}

}  // namespace

void mlog_free(MetricsLog* m) {
  if (m->ring) cudaFree(m->ring);
  if (m->h_rows) cudaFreeHost(m->h_rows);
  if (m->h_step) cudaFreeHost(m->h_step);
  *m = MetricsLog{};
}

int mlog_enable(MetricsLog* m, int cap, int K, const long long* d_step, cudaStream_t s) {
  if (cap < 0 || K < 1 || K > MLOG_MAX_K) return b2g_fail(B2G_EINVAL, "metrics log: capacity must be >= 0");
  CK(cudaStreamSynchronize(s));       // no step still writes into the ring that is freed here
  mlog_free(m);
  if (cap == 0) return 0;
  const size_t bytes = (size_t)cap * K * sizeof(float);
  if (cudaMalloc((void**)&m->ring, bytes) != cudaSuccess || cudaMallocHost((void**)&m->h_rows, bytes) != cudaSuccess ||
      cudaMallocHost((void**)&m->h_step, sizeof(long long)) != cudaSuccess) {
    cudaGetLastError();
    mlog_free(m);
    return b2g_fail(B2G_ECUDA, "metrics log: allocation of " + std::to_string(cap) + " rows failed");
  }
  m->cap = cap; m->K = K;
  return mlog_rebase(m, d_step, s);
}

int mlog_rebase(MetricsLog* m, const long long* d_step, cudaStream_t s) {
  if (!m->on()) return 0;
  return read_step(m, d_step, s, &m->drained);
}

void mlog_append(const MetricsLog& m, const MetricsLogSrc& src, const long long* d_step, cudaStream_t s) {
  metrics_log_append_kernel<<<1, 32, 0, s>>>(m.ring, m.cap, m.K, d_step, src);
}

int mlog_drain(MetricsLog* m, const long long* d_step, cudaStream_t s, float* rows, int max_rows, int64_t* first_step,
               int* n_rows, int64_t* lost, const std::function<void(float*)>& fix) {
  if (!m->on()) return b2g_fail(B2G_ESTATE, "metrics log is off: enable it with b2g_*_metrics_log(h, capacity)");
  if (max_rows < 0 || (max_rows > 0 && !rows)) return b2g_fail(B2G_EINVAL, "metrics drain: bad rows / max_rows");
  long long cur = 0;
  if (int rc = read_step(m, d_step, s, &cur)) return rc;
  if (cur < m->drained) m->drained = cur;
  const long long avail = cur - m->drained;
  const long long dropped = std::max(0LL, avail - (long long)m->cap);
  const long long start = m->drained + dropped;
  const int n = (int)std::min<long long>(avail - dropped, max_rows);
  const int K = m->K;
  if (n > 0) {
    const long long p0 = start % m->cap;
    const long long n0 = std::min<long long>(n, m->cap - p0);
    CK(cudaMemcpyAsync(m->h_rows, m->ring + p0 * K, (size_t)n0 * K * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (n > n0) CK(cudaMemcpyAsync(m->h_rows + n0 * K, m->ring, (size_t)(n - n0) * K * sizeof(float), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    for (int r = 0; r < n; ++r) {
      float* row = m->h_rows + (size_t)r * K;
      if (fix) fix(row);
      memcpy(rows + (size_t)r * K, row, K * sizeof(float));
    }
  }
  m->drained = start + n;
  if (first_step) *first_step = start + 1;
  if (n_rows) *n_rows = n;
  if (lost) *lost = dropped;
  return 0;
}

}  // namespace b2g
