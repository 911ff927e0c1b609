// Optimiser + bookkeeping kernels: HBM/L2-bound, 128-bit vectorised, one pass over the arenas.
//
//  * prep_kernel  : head of every step -- advances the three Adam step counters, evaluates the TF1
//                   bias-corrected step size lr_t = lr*sqrt(1-b2^t)/(1-b1^t) (tf.train.AdamOptimizer),
//                   zeroes the metric accumulators and draws replay indices (ReplayBuffer.sample:
//                   random.randint) and N(0,1) policy noise (tf.random_normal) from Philox4x32-10.
//  * optim_kernel : policy Adam -> values Adam -> entropy Adam ([SB2] sac.py control-dependency
//                   order; they touch disjoint variables so one fused pass is equivalent), then the
//                   Polyak target update theta_T <- (1-tau) theta_T + tau theta_V on the UPDATED
//                   values_fn ([SB2] target_update_op), plus squared gradient norms per optimiser.
#include <math.h>

#include <cuda_bf16.h>

#include "common.cuh"

namespace b2g {
namespace {

__device__ __forceinline__ float u01(unsigned x) { return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f); }

__global__ void prep_kernel(PrepArgs a) {
  const int tid = threadIdx.x;
  __shared__ long long s_rng;
  if (tid == 0) {
    s_rng = a.counters[4];
    if (a.apply) {
      const double lr = (double)a.lr[0];
      for (int g = 0; g < 3; ++g) {
        const long long t = ++a.counters[g];
        a.step_consts[g] = lr * sqrt(1.0 - pow(0.999, (double)t)) / (1.0 - pow(0.9, (double)t));
      }
      a.counters[3] += 1;
    }
    if (a.gen && !a.defer_bump) a.counters[4] += 1;
  }
  if (tid < MET_COUNT) a.metrics[tid] = 0.f;
  __syncthreads();
  if (!a.gen) return;
  const unsigned long long step = (unsigned long long)s_rng;
  const uint2 key = make_uint2((unsigned)a.seed, (unsigned)(a.seed >> 32));
  // stream 0: replay indices; stream 1: policy noise
  const unsigned long long rsz = (unsigned long long)(a.replay_size ? a.replay_size[0] : a.counters[5]);
  for (int i = tid; i < (a.skip_indices ? 0 : (a.B + 3) / 4); i += blockDim.x) {
    const uint4 r = philox4x32_10(make_uint4((unsigned)step, (unsigned)(step >> 32), (unsigned)i, 0u), key);
    const unsigned v[4] = {r.x, r.y, r.z, r.w};
    for (int j = 0; j < 4; ++j) {
      const int b = 4 * i + j;
      if (b >= a.B) continue;
      const int u = (int)(((unsigned long long)v[j] * rsz) >> 32);
      a.indices[b] = a.ring_cap > 0 ? ring_slot(a.counters[6], u, a.ring_cap) : u;
    }
  }
  const int n_eps = a.B * a.A;
  for (int i = tid; i < (n_eps + 3) / 4; i += blockDim.x) {
    const uint4 r = philox4x32_10(make_uint4((unsigned)step, (unsigned)(step >> 32), (unsigned)i, 1u), key);
    const float r0 = sqrtf(-2.f * logf(u01(r.x))), r1 = sqrtf(-2.f * logf(u01(r.z)));
    float s0, c0, s1, c1;
    sincospif(2.f * u01(r.y), &s0, &c0);
    sincospif(2.f * u01(r.w), &s1, &c1);
    const float z[4] = {r0 * c0, r0 * s0, r1 * c1, r1 * s1};
    for (int j = 0; j < 4; ++j)
      if (4 * i + j < n_eps) a.eps[4 * i + j] = z[j];
  }
}

__global__ void __launch_bounds__(256) optim_kernel(OptimArgs a) {
  const int n_total4 = (a.n_pi + a.n_values + a.n_ent) >> 2;
  const float b1 = 0.9f, b2 = 0.999f, eps = 1e-8f;
  const float lrt[3] = {(float)a.step_consts[0], (float)a.step_consts[1], (float)a.step_consts[2]};
  float ss[2] = {0.f, 0.f};
  const bool ranged = a.r_hi[0] > 0 || a.r_hi[1] > 0;
  const int len0 = ranged ? (a.r_hi[0] - a.r_lo[0]) >> 2 : n_total4, len1 = ranged ? (a.r_hi[1] - a.r_lo[1]) >> 2 : 0;
  for (int k4 = blockIdx.x * blockDim.x + threadIdx.x; k4 < len0 + len1; k4 += gridDim.x * blockDim.x) {
    const int i4 = !ranged ? k4 : (k4 < len0 ? (a.r_lo[0] >> 2) + k4 : (a.r_lo[1] >> 2) + (k4 - len0));
    const int i = i4 << 2;
    const int grp = i < a.n_pi ? 0 : (i < a.n_pi + a.n_values ? 1 : 2);
    float4 g = reinterpret_cast<const float4*>(a.G)[i4];
    g.x *= a.grad_scale; g.y *= a.grad_scale; g.z *= a.grad_scale; g.w *= a.grad_scale;
    const float s2 = g.x * g.x + g.y * g.y + g.z * g.z + g.w * g.w;
    if (grp < 2) ss[grp] += s2;
    if (!a.apply) continue;
    float4 m = reinterpret_cast<float4*>(a.Mo)[i4], v = reinterpret_cast<float4*>(a.Vo)[i4];
    float4 p = reinterpret_cast<float4*>(a.P)[i4];
    const float lr = lrt[grp];
#define B2G_ADAM(c)                                   \
  m.c = b1 * m.c + (1.f - b1) * g.c;                  \
  v.c = b2 * v.c + (1.f - b2) * (g.c * g.c);          \
  p.c = p.c - lr * m.c / (sqrtf(v.c) + eps);
    B2G_ADAM(x) B2G_ADAM(y) B2G_ADAM(z) B2G_ADAM(w)
#undef B2G_ADAM
    reinterpret_cast<float4*>(a.Mo)[i4] = m;
    reinterpret_cast<float4*>(a.Vo)[i4] = v;
    reinterpret_cast<float4*>(a.P)[i4] = p;
    const int j = i - a.n_pi;
    if (grp == 1 && j < a.n_target) {
      float4 tg = reinterpret_cast<float4*>(a.T)[j >> 2];
      const float tau = a.tau, om = 1.f - a.tau;
      tg.x = om * tg.x + tau * p.x; tg.y = om * tg.y + tau * p.y;
      tg.z = om * tg.z + tau * p.z; tg.w = om * tg.w + tau * p.w;
      reinterpret_cast<float4*>(a.T)[j >> 2] = tg;
    }
  }
  // block reduce of the two squared norms
  __shared__ float red[2][8];
  for (int k = 0; k < 2; ++k) {
    float v = ss[k];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  if (threadIdx.x < 2) {
    float v = 0.f;
    for (int w = 0; w < 8; ++w) v += red[threadIdx.x][w];
    atomicAdd(a.metrics + MET_GN_PI + threadIdx.x, v);
  }
  if (a.bump_counter && blockIdx.x == 0 && threadIdx.x == 0) *a.bump_counter += 1;
}

// weights -> BF16 hi/lo planes; 32x32 smem-tiled transpose for the [N,R] copy (both sides coalesced)
__global__ void __launch_bounds__(256) planes_kernel(const PlaneJob* __restrict__ jobs, int njobs) {
  __shared__ float tile[32][33];
  int j = 0;
  while (j + 1 < njobs && (int)blockIdx.x >= jobs[j + 1].tile_start) ++j;
  const PlaneJob job = jobs[j];
  const int t = blockIdx.x - job.tile_start;
  const int tiles_n = (job.N + 31) / 32;
  const int r0 = (t / tiles_n) * 32, n0 = (t % tiles_n) * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;     // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int r = r0 + i, n = n0 + tx;
    float v = 0.f;
    if (r < job.R && n < job.N) {
      v = job.src[(size_t)r * job.N + n];
      if (job.hi) {
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        job.hi[(size_t)r * job.N + n] = __bfloat16_as_ushort(h);
        job.lo[(size_t)r * job.N + n] = __bfloat16_as_ushort(__float2bfloat16_rn(v - __bfloat162float(h)));
      }
    }
    tile[i][tx] = v;
  }
  __syncthreads();
  if (job.hiT) {
    for (int i = ty; i < 32; i += 8) {
      const int n = n0 + i, r = r0 + tx;
      if (r < job.R && n < job.N) {
        const float v = tile[tx][i];
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        job.hiT[(size_t)n * job.R + r] = __bfloat16_as_ushort(h);
        job.loT[(size_t)n * job.R + r] = __bfloat16_as_ushort(__float2bfloat16_rn(v - __bfloat162float(h)));
      }
    }
  }
}

// bias gradients as column sums of the (masked) gradient maps.  Thread = (row group, float4 column group);
// 8 rows per thread, all table + data loads of a thread issued as one batch; block reduce, then N atomics.
__global__ void __launch_bounds__(256) colsum_kernel(const ColsumJob* __restrict__ jobs, int njobs) {
  __shared__ float red[512];
  int j = 0;
  while (j + 1 < njobs && (int)blockIdx.x >= jobs[j + 1].cta_start) ++j;
  const ColsumJob job = jobs[j];
  const int N = job.N, N4 = N >> 2, tid = threadIdx.x;
  const int groups = 256 / N4;                 // N <= 1024
  const int rows_per_cta = 8 * groups;
  const int r0 = (blockIdx.x - job.cta_start) * rows_per_cta;
  for (int i = tid; i < N; i += 256) red[i] = 0.f;
  __syncthreads();
  const int g = tid / N4, c4 = tid - g * N4;
  if (g < groups) {
    int off[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = r0 + g + i * groups;
      off[i] = r < job.rows ? job.row_off[r] : -1;
    }
    float4 s = make_float4(0, 0, 0, 0);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (off[i] >= 0) {
        const float4 v = *reinterpret_cast<const float4*>(job.src + off[i] + 4 * c4);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      }
    }
    atomicAdd(&red[4 * c4 + 0], s.x); atomicAdd(&red[4 * c4 + 1], s.y);
    atomicAdd(&red[4 * c4 + 2], s.z); atomicAdd(&red[4 * c4 + 3], s.w);
  }
  __syncthreads();
  for (int i = tid; i < N; i += 256) atomicAdd(job.dst + i, red[i]);
}
}  // namespace

void colsum_launch(const ColsumJob* dev_jobs, int njobs, int total_ctas, cudaStream_t s) {
  if (total_ctas > 0) colsum_kernel<<<total_ctas, 256, 0, s>>>(dev_jobs, njobs);
}

void planes_launch(const PlaneJob* dev_jobs, int njobs, int total_tiles, cudaStream_t s) {
  if (total_tiles > 0) planes_kernel<<<total_tiles, 256, 0, s>>>(dev_jobs, njobs);
}

void prep_launch(const PrepArgs& a, cudaStream_t s) { prep_kernel<<<1, 256, 0, s>>>(a); }

namespace {
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ long long gtime() { long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ void st_release_sys(int* p, int v) { asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

// All cross-GPU traffic is STORES (posted, ~3x the throughput of peer loads measured here: tools/dp_trace.py): every rank first pushes
// the slices of its gradient buffer it does not own into the owners' receive arenas, the owners then read only local memory.
// One CTA per SM (all resident: phases A and B are separated by a grid-wide arrival counter and by flags from the other GPUs).
template <int NR>
__global__ void __launch_bounds__(1024) dp_optim_kernel(DpArgs d) {
  const OptimArgs& a = d.o;
  const int N = d.nranks, me = d.rank, tid = threadIdx.x;
  const int epoch = (int)d.counters[3];
  // exchange block of a rank (ints): [0,8) "gradients of rank q have landed here", [8,16) "slice of rank q written here", [16,32)
  // squared-norm partials part[q][2], [32,160) loss scalars loss[q][16]
  int* xl = d.x_peer[me];
  long long* stamp = reinterpret_cast<long long*>(d.sync + 8);      // bring-up: %globaltimer at the phase boundaries (tools/dp_trace.py)
  if (blockIdx.x == 0 && tid == 0) stamp[0] = gtime();
  const int n_train4 = (a.n_pi + a.n_values + a.n_ent) >> 2;
  const int per4 = (n_train4 + N - 1) / N, lo4 = me * per4, hi4 = min(n_train4, lo4 + per4);
  const int nthr = gridDim.x * blockDim.x, gtid = blockIdx.x * blockDim.x + tid;
  __shared__ int s_last;
  // ---- A. push: slice q of my gradients -> receive arena of rank q, row `me`; my loss scalars -> everybody's exchange block
  for (int q = 0; q < N; ++q) {
    if (q == me) continue;
    const int qlo = q * per4, qhi = min(n_train4, qlo + per4);
    float4* dst = reinterpret_cast<float4*>(d.R_peer[q]) + (size_t)me * per4;
    const float4* src = reinterpret_cast<const float4*>(a.G);
    for (int i4 = qlo + gtid; i4 < qhi; i4 += nthr) {
      if ((i4 >= d.skip_lo4[0] && i4 < d.skip_hi4[0]) || (i4 >= d.skip_lo4[1] && i4 < d.skip_hi4[1])) continue;   // pushed by the cnn_fc1 wgrad epilogue
      dst[i4 - qlo] = __ldcs(src + i4);
    }
  }
  if (blockIdx.x == 0 && tid < N * MET_GN_PI) {
    const int q = tid / MET_GN_PI, k = tid - q * MET_GN_PI;
    reinterpret_cast<float*>(d.x_peer[q] + 32)[me * 16 + k] = a.metrics[k];
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence_system();                        // this CTA's peer stores before its arrival
    s_last = atomicAdd(d.sync, 1) == (int)gridDim.x - 1;
  }
  __syncthreads();
  if (s_last && tid < N) { __threadfence_system(); st_release_sys(d.x_peer[tid] + me, epoch); }   // everything of mine has landed
  if (tid < N) { while (ld_acquire_sys(xl + tid) < epoch) __nanosleep(100); }
  __syncthreads();
  if (blockIdx.x == 0 && tid == 0) stamp[1] = gtime();
  if (blockIdx.x == 0 && tid < MET_GN_PI) {        // loss scalars: sums in fixed rank order, identical on every rank
    const float* loss = reinterpret_cast<const float*>(xl + 32);
    float v = 0.f;
    for (int q = 0; q < N; ++q) v += __ldcg(loss + q * 16 + tid);
    a.metrics[tid] = v;
  }
  // ---- B. my slice: sum the N copies (mine from the gradient buffer, the others from my receive arena; fixed rank order: every
  //         replica of a parameter sees the same sum), Adam / Polyak, push the new values into every replica
  const float b1 = 0.9f, b2 = 0.999f, eps = 1e-8f;
  const float lrt[3] = {(float)a.step_consts[0], (float)a.step_consts[1], (float)a.step_consts[2]};
  float ss[2] = {0.f, 0.f};
  const float4* R = reinterpret_cast<const float4*>(d.R_peer[me]);
  for (int i4 = lo4 + gtid; i4 < hi4; i4 += nthr) {
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int q = 0; q < NR; ++q)
      if (q < N) {
        const float4 v = q == me ? reinterpret_cast<const float4*>(a.G)[i4] : __ldcg(R + (size_t)q * per4 + (i4 - lo4));
        g.x += v.x; g.y += v.y; g.z += v.z; g.w += v.w;
      }
    const int i = i4 << 2;
    const int grp = i < a.n_pi ? 0 : (i < a.n_pi + a.n_values ? 1 : 2);
    g.x *= a.grad_scale; g.y *= a.grad_scale; g.z *= a.grad_scale; g.w *= a.grad_scale;
    if (grp < 2) ss[grp] += g.x * g.x + g.y * g.y + g.z * g.z + g.w * g.w;
    float4 m = reinterpret_cast<float4*>(a.Mo)[i4], v = reinterpret_cast<float4*>(a.Vo)[i4];
    float4 p = reinterpret_cast<float4*>(a.P)[i4];
    const float lr = lrt[grp];
#define B2G_ADAM(c)                                   \
  m.c = b1 * m.c + (1.f - b1) * g.c;                  \
  v.c = b2 * v.c + (1.f - b2) * (g.c * g.c);          \
  p.c = p.c - lr * m.c / (sqrtf(v.c) + eps);
    B2G_ADAM(x) B2G_ADAM(y) B2G_ADAM(z) B2G_ADAM(w)
#undef B2G_ADAM
    reinterpret_cast<float4*>(a.Mo)[i4] = m;
    reinterpret_cast<float4*>(a.Vo)[i4] = v;
    for (int q = 0; q < N; ++q) reinterpret_cast<float4*>(d.P_peer[q])[i4] = p;
    const int j = i - a.n_pi;
    if (grp == 1 && j < a.n_target) {
      const int t4 = n_train4 + (j >> 2);         // target block sits behind the trainable arena
      float4 tg = reinterpret_cast<float4*>(a.P)[t4];
      const float tau = a.tau, om = 1.f - a.tau;
      tg.x = om * tg.x + tau * p.x; tg.y = om * tg.y + tau * p.y;
      tg.z = om * tg.z + tau * p.z; tg.w = om * tg.w + tau * p.w;
      for (int q = 0; q < N; ++q) reinterpret_cast<float4*>(d.P_peer[q])[t4] = tg;
    }
  }
  if (blockIdx.x == 0 && tid == 0) stamp[2] = gtime();
  // ---- C. squared gradient norms of my slice, then: the last CTA publishes them and "my slice is written everywhere"
  __shared__ float red[2][32];
  for (int k = 0; k < 2; ++k) {
    float v = ss[k];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((tid & 31) == 0) red[k][tid >> 5] = v;
  }
  __syncthreads();
  float* acc = reinterpret_cast<float*>(d.sync + 2);
  if (tid < 2) {
    float v = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v += red[tid][w];
    atomicAdd(acc + tid, v);
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence_system();
    s_last = atomicAdd(d.sync + 1, 1) == (int)gridDim.x - 1;
  }
  __syncthreads();
  if (!s_last) return;
  if (tid == 0) stamp[3] = gtime();
  __threadfence();
  if (tid < N) {
    float* part = reinterpret_cast<float*>(d.x_peer[tid] + 16) + 2 * me;
    part[0] = __ldcg(acc); part[1] = __ldcg(acc + 1);
    __threadfence_system();
    st_release_sys(d.x_peer[tid] + 8 + me, epoch);
  }
  if (tid < N) { while (ld_acquire_sys(xl + 8 + tid) < epoch) __nanosleep(100); }
  __syncthreads();
  if (tid < 2) {                                   // fixed order again: identical metrics on every rank
    const float* part = reinterpret_cast<const float*>(xl + 16);
    float v = 0.f;
    for (int q = 0; q < N; ++q) v += __ldcg(part + 2 * q + tid);
    a.metrics[MET_GN_PI + tid] += v;
  }
  if (tid == 0) {
    stamp[4] = gtime();
    d.sync[0] = 0; d.sync[1] = 0; acc[0] = 0.f; acc[1] = 0.f;
    if (a.bump_counter) *a.bump_counter += 1;
  }
}
}  // namespace

void dp_optim_launch(const DpArgs& a, int ctas, cudaStream_t s) {
  if (a.nranks <= 2) dp_optim_kernel<2><<<ctas, 1024, 0, s>>>(a);
  else if (a.nranks <= 4) dp_optim_kernel<4><<<ctas, 1024, 0, s>>>(a);
  else dp_optim_kernel<8><<<ctas, 1024, 0, s>>>(a);
}

void optim_launch(const OptimArgs& a, cudaStream_t s) {
  int n4 = (a.n_pi + a.n_values + a.n_ent) >> 2;
  if (a.r_hi[0] > 0 || a.r_hi[1] > 0) n4 = ((a.r_hi[0] - a.r_lo[0]) + (a.r_hi[1] - a.r_lo[1])) >> 2;
  if (n4 <= 0) return;
  int grid = (n4 + 255) / 256;
  if (grid > 132 * 8) grid = 132 * 8;
  optim_kernel<<<grid, 256, 0, s>>>(a);
}

}  // namespace b2g
