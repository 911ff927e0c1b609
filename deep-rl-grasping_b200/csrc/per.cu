// Prioritised-replay kernels (declarations and the tree layout in per.cuh).
#include <math.h>

#include "common.cuh"
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

}  // namespace b2g
