// Prioritised-replay kernels and the transition replay (declarations and the tree layout in per.cuh).
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "host.cuh"
#include "per.cuh"

namespace b2g {
namespace {

// one CTA, B threads: draws B slots proportionally to priority (find_prefixsum_idx descent) and their IS weights
__global__ void per_sample_kernel(PerArgs a) {
  const int b = threadIdx.x;
  if (b >= a.B) return;
  const unsigned long long step = (unsigned long long)a.counters[4];
  const long long size = a.counters[5];
  const uint4 r = philox4x32_10(make_uint4((unsigned)step, (unsigned)(step >> 32), (unsigned)(b >> 2), 2u), make_uint2((unsigned)a.seed, (unsigned)(a.seed >> 32)));
  const unsigned v = (b & 3) == 0 ? r.x : (b & 3) == 1 ? r.y : (b & 3) == 2 ? r.z : r.w;
  const double total = a.tsum[1];
  double mass = ((double)v + 0.5) * (1.0 / 4294967296.0) * total;
  long long node = 1;
  while (node < a.C) {
    const double left = a.tsum[2 * node];
    if (left > mass) node = 2 * node;
    else { mass -= left; node = 2 * node + 1; }
  }
  long long idx = node - a.C;
  if (idx >= size) idx = size - 1;                       // (rounding at the right edge of the occupied range)
  const double beta = (double)a.beta[0];
  const double p_min = a.tmin[1] / total;
  const double max_w = pow(p_min * (double)size, -beta);
  const double p = a.tsum[a.C + idx] / total;
  a.indices[b] = (int)idx;
  a.weights[b] = (float)(pow(p * (double)size, -beta) / max_w);
}

// one CTA: writes `n` leaves and repairs their ancestors level by level (siblings recomputed redundantly: same values)
__global__ void per_write_kernel(PerArgs a, const int* __restrict__ slots, long long first_slot, long long cap, int n, int from_td) {
  const int i = threadIdx.x;
  long long leaf = 0;
  if (i < n) {
    const long long slot = slots ? (long long)slots[i] : (first_slot + i) % cap;
    float raw;
    if (from_td) {
      float s = 0.f;
      for (int d = 0; d < a.D; ++d) s += fabsf(a.td[i * a.D + d]);
      raw = s + a.eps;
      atomicMax(reinterpret_cast<int*>(a.max_prio), __float_as_int(raw));      // positive floats order like their bit patterns
      if (a.prio_out) a.prio_out[i] = raw;
    } else raw = a.max_prio[0];
    const double pr = pow((double)raw, (double)a.alpha);
    leaf = a.C + slot;
    a.tsum[leaf] = pr; a.tmin[leaf] = pr;
  }
  __syncthreads();
  for (long long span = a.C; span > 1; span >>= 1) {
    if (i < n) {
      leaf >>= 1;
      a.tsum[leaf] = a.tsum[2 * leaf] + a.tsum[2 * leaf + 1];
      a.tmin[leaf] = fmin(a.tmin[2 * leaf], a.tmin[2 * leaf + 1]);
    }
    __syncthreads();
  }
}

__global__ void per_init_kernel(double* tsum, double* tmin, long long n2, float* max_prio) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n2; i += (long long)gridDim.x * blockDim.x) { tsum[i] = 0.0; tmin[i] = INFINITY; }
  if (blockIdx.x == 0 && threadIdx.x == 0) max_prio[0] = 1.0f;
}

}  // namespace

void per_sample_launch(const PerArgs& a, cudaStream_t s) { per_sample_kernel<<<1, ((a.B + 31) / 32) * 32, 0, s>>>(a); }

void per_write_launch(const PerArgs& a, const int* slots, long long first_slot, long long cap, int n, int from_td, cudaStream_t s) {
  per_write_kernel<<<1, ((n + 31) / 32) * 32, 0, s>>>(a, slots, first_slot, cap, n, from_td);
}

void per_init_launch(double* tsum, double* tmin, long long n2, float* max_prio, cudaStream_t s) {
  per_init_kernel<<<256, 256, 0, s>>>(tsum, tmin, n2, max_prio);
}

int TransitionReplay::init(std::vector<void*>& allocs, cudaStream_t s, int64_t cap_, int E_, int A_, int B, bool per_, float alpha_,
                           float eps_) {
  cap = cap_; E = E_; A = A_; per = per_; alpha = alpha_; eps = eps_;
  if (int rc = dev_alloc(allocs, s, &obs, cap * E)) return rc;
  if (int rc = dev_alloc(allocs, s, &next, cap * E)) return rc;
  if (int rc = dev_alloc(allocs, s, &act, cap * A)) return rc;
  if (int rc = dev_alloc(allocs, s, &rew, cap)) return rc;
  if (int rc = dev_alloc(allocs, s, &done, cap)) return rc;
  if (int rc = dev_alloc(allocs, s, &beta, 1)) return rc;
  if (int rc = dev_alloc(allocs, s, &max_prio, 1)) return rc;
  if (int rc = dev_alloc(allocs, s, &prio_out, B)) return rc;
  if (!per) return 0;
  per_C = 1;
  while (per_C < cap) per_C <<= 1;
  if (int rc = dev_alloc(allocs, s, &t_sum, 2 * per_C)) return rc;
  if (int rc = dev_alloc(allocs, s, &t_min, 2 * per_C)) return rc;
  per_init_launch(t_sum, t_min, 2 * per_C, max_prio, s);
  const float beta0 = 0.4f;
  CK(cudaMemcpyAsync(beta, &beta0, sizeof(float), cudaMemcpyHostToDevice, s));
  return 0;
}

PerArgs TransitionReplay::per_args(const long long* counters, unsigned long long seed, int B, int* indices, float* weights, const float* td,
                                   int D) const {
  PerArgs pr{};
  pr.tsum = t_sum; pr.tmin = t_min; pr.C = per_C; pr.max_prio = max_prio; pr.counters = counters; pr.seed = seed;
  pr.B = B; pr.alpha = alpha; pr.eps = eps; pr.beta = beta; pr.indices = indices; pr.weights = weights;
  pr.prio_out = prio_out; pr.td = td; pr.D = D;
  return pr;
}

void TransitionReplay::insert_max_prio(int64_t first, int64_t n, cudaStream_t s) const {
  if (!per) return;
  const PerArgs pr = per_args(nullptr, 0, 0, nullptr, nullptr, nullptr, 0);
  for (int64_t o = 0; o < n; o += 1024) per_write_launch(pr, nullptr, first + o, cap, (int)std::min<int64_t>(1024, n - o), 0, s);
}

void TransitionReplay::advance(int64_t n) {
  pos = (pos + n) % cap;
  size = std::min(cap, size + n);
}

int TransitionReplay::add(const float* o, const float* a, const float* r, const float* nx, const float* d, int64_t n, long long* counters,
                          cudaStream_t s) {
  for (int64_t done_n = 0; done_n < n;) {
    const int64_t chunk = std::min(n - done_n, cap - pos);
    CK(cudaMemcpyAsync(obs + pos * E, o + done_n * E, chunk * E * sizeof(float), cudaMemcpyDefault, s));
    CK(cudaMemcpyAsync(next + pos * E, nx + done_n * E, chunk * E * sizeof(float), cudaMemcpyDefault, s));
    CK(cudaMemcpyAsync(act + pos * A, a + done_n * A, chunk * A * sizeof(float), cudaMemcpyDefault, s));
    CK(cudaMemcpyAsync(rew + pos, r + done_n, chunk * sizeof(float), cudaMemcpyDefault, s));
    CK(cudaMemcpyAsync(done + pos, d + done_n, chunk * sizeof(float), cudaMemcpyDefault, s));
    insert_max_prio(pos, chunk, s);
    advance(chunk);
    done_n += chunk;
  }
  const long long sz = size;
  CK(cudaMemcpyAsync(counters + 5, &sz, sizeof(long long), cudaMemcpyHostToDevice, s));
  CK(cudaStreamSynchronize(s));
  return 0;
}

int TransitionReplay::set_beta(float b, int device, cudaStream_t s) {
  CK(cudaSetDevice(device));
  CK(cudaStreamSynchronize(s));
  CK(cudaMemcpy(beta, &b, sizeof(float), cudaMemcpyHostToDevice));
  return 0;
}

int TransitionReplay::get_last(const int* indices, const float* weights, int B, int32_t* slots, float* w, float* p, int device,
                               cudaStream_t s) const {
  CK(cudaSetDevice(device));
  CK(cudaStreamSynchronize(s));
  if (slots) CK(cudaMemcpy(slots, indices, B * sizeof(int32_t), cudaMemcpyDeviceToHost));
  if (w) CK(cudaMemcpy(w, weights, B * sizeof(float), cudaMemcpyDeviceToHost));
  if (p) CK(cudaMemcpy(p, prio_out, B * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

std::vector<StateSection> TransitionReplay::state_sections(int64_t live) const {
  const size_t fb = sizeof(float);
  std::vector<StateSection> s(7);
  s[0].tag = state_tag("ROBS"); s[0].pieces = {dev_piece(obs, live * E * fb)};
  s[1].tag = state_tag("RNXT"); s[1].pieces = {dev_piece(next, live * E * fb)};
  s[2].tag = state_tag("RACT"); s[2].pieces = {dev_piece(act, cap * A * fb)};
  s[3].tag = state_tag("RREW"); s[3].pieces = {dev_piece(rew, cap * fb)};
  s[4].tag = state_tag("RDON"); s[4].pieces = {dev_piece(done, cap * fb)};
  s[5].tag = state_tag("PERT");
  if (per) s[5].pieces = {dev_piece(t_sum, 2 * per_C * sizeof(double)), dev_piece(t_min, 2 * per_C * sizeof(double))};
  s[6].tag = state_tag("PERS"); s[6].pieces = {dev_piece(max_prio, sizeof(float)), dev_piece(beta, sizeof(float))};
  return s;
}

}  // namespace b2g
