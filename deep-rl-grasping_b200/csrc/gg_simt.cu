// fp32 CUDA-core gather-GEMM engine (precision mode B2G_PREC_FP32_SIMT).
//
// Bit-faithful fp32 FFMA arithmetic for every dense contraction on the SAC step; it is the
// on-device numerical reference the wgmma engine (gg_tc.cu) is validated against, and the
// engine used for the small head-side contractions in every mode.
// Tile: 64(m) x 64(n) x 16(r), 256 threads, 4x4 outputs per thread, register-prefetched smem.
#include <cuda_bf16.h>

#include <type_traits>

#include "common.cuh"

namespace b2g {
namespace {
constexpr int BM = GG_SIMT_BM, BN = GG_SIMT_BN, BK = GG_SIMT_BK, PAD = 4;

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }

// EXT: the auto-encoder's variant, which adds element-wise m-contiguous A gathers (GG_A_SCALAR without GG_A_RVEC) and the
// GG_EPI_LRELU_GRAD epilogue, and sums in double: fp32 products are exact in double, so a long reduction whose terms cancel
// (a weight or bias gradient over every pixel of a batch) keeps its accuracy; its GG_EPI_ATOMIC and GG_COLSUM destinations
// are double arrays (C and colsum reinterpreted), accumulated without rounding to fp32.  The plain instantiation is the
// engine every other path launches, unchanged.
// TANH: the PPO variant (fp32 sums, as the plain engine), which adds GG_EPI_BIAS_TANH and GG_EPI_TANH_GRAD (ppo.cu).
template <bool EXT, bool TANH>
__device__ __forceinline__ void gg_simt_body(const GemmDesc* __restrict__ descs, int ndesc) {
  __shared__ GemmDesc sd;
  __shared__ __align__(16) float As[BK][BM + PAD];
  __shared__ __align__(16) float Bs[BK][BN + PAD];
  using Acc = typename std::conditional<EXT, double, float>::type;
  __shared__ Acc cs[BN];
  const int tid = threadIdx.x;
  if (tid == 0) {
    int p = 0;
    const int t = blockIdx.x;
    while (p + 1 < ndesc && t >= descs[p + 1].tile_start) ++p;
    sd = descs[p];
  }
  if (tid < BN) cs[tid] = 0;
  pdl_trigger();
  pdl_wait();
  __syncthreads();
  const GemmDesc& d = sd;
  int t = blockIdx.x - d.tile_start;
  const int per = d.tiles_m * d.tiles_n;
  const int split = t / per;
  t -= split * per;
  const int tm = t / d.tiles_n, tn = t - tm * d.tiles_n;
  const int m0 = tm * BM, n0 = tn * BN;
  const int chunk = (((d.R + d.splitR - 1) / d.splitR) + BK - 1) / BK * BK;
  const int r_begin = split * chunk;
  const int r_end = min(d.R, r_begin + chunk);
  const bool a_rvec = d.flags & GG_A_RVEC, b_rvec = d.flags & GG_B_RVEC;
  const bool do_colsum = (d.flags & GG_COLSUM) && tm == 0;
  const bool a_scalar = d.flags & GG_A_SCALAR;
  const float* __restrict__ A = d.A;
  const float* __restrict__ Bp = d.B;

  // ---- per-thread load coordinates
  // A, r-contiguous: (m = tid/4, r4 = (tid%4)*4); A, m-contiguous: (r = tid/16, m4 = (tid%16)*4)
  const int a_m = a_rvec ? (tid >> 2) : ((tid & 15) << 2);
  const int a_r = a_rvec ? ((tid & 3) << 2) : (tid >> 4);
  int a_off[4];   // m-side offsets (rvec: one; mvec: base of the group)
  bool a_ok[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { a_ok[i] = false; a_off[i] = 0; }
  if (a_rvec) {
    a_ok[0] = (m0 + a_m) < d.M;
    a_off[0] = a_ok[0] ? d.aM[m0 + a_m] : 0;
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      a_ok[i] = (m0 + a_m + i) < d.M;
      a_off[i] = a_ok[i] ? d.aM[m0 + a_m + i] : 0;
    }
  }
  const int b_n = b_rvec ? (tid >> 2) : ((tid & 15) << 2);
  const int b_r = b_rvec ? ((tid & 3) << 2) : (tid >> 4);
  int b_off[4];
  bool b_ok[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { b_ok[i] = false; b_off[i] = 0; }
  if (b_rvec) {
    b_ok[0] = (n0 + b_n) < d.N;
    b_off[0] = b_ok[0] ? d.bN[n0 + b_n] : 0;
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      b_ok[i] = (n0 + b_n + i) < d.N;
      b_off[i] = b_ok[i] ? d.bN[n0 + b_n + i] : 0;
    }
  }

  float4 ra = make_float4(0, 0, 0, 0), rb = make_float4(0, 0, 0, 0);
  Acc csum[4] = {0, 0, 0, 0};

  auto load_tiles = [&](int rk) {
    // ---- A
    if (a_rvec) {
      const int r = rk + a_r;
      ra = make_float4(0, 0, 0, 0);
      if (a_ok[0] && r < r_end) {
        if (r + 3 < r_end && !a_scalar) {
          ra = ld4(A + a_off[0] + d.aR[r]);
        } else {
          float v[4] = {0, 0, 0, 0};
          for (int i = 0; i < 4; ++i)
            if (r + i < r_end) v[i] = A[a_off[0] + d.aR[r + i]];
          ra = make_float4(v[0], v[1], v[2], v[3]);
        }
      }
    } else {
      const int r = rk + a_r;
      ra = make_float4(0, 0, 0, 0);
      if (r < r_end) {
        const int ar = d.aR[r];
        if (a_ok[3] && !(EXT && a_scalar)) {
          ra = ld4(A + a_off[0] + ar);
        } else {
          float v[4] = {0, 0, 0, 0};
#pragma unroll
          for (int i = 0; i < 4; ++i)
            if (a_ok[i]) v[i] = A[a_off[i] + ar];
          ra = make_float4(v[0], v[1], v[2], v[3]);
        }
      }
    }
    // ---- B
    if (b_rvec) {
      const int r = rk + b_r;
      rb = make_float4(0, 0, 0, 0);
      if (b_ok[0] && r < r_end) {
        if (r + 3 < r_end) {
          rb = ld4(Bp + b_off[0] + d.bR[r]);
        } else {
          float v[4] = {0, 0, 0, 0};
          for (int i = 0; i < 4; ++i)
            if (r + i < r_end) v[i] = Bp[b_off[0] + d.bR[r + i]];
          rb = make_float4(v[0], v[1], v[2], v[3]);
        }
      }
    } else {
      const int r = rk + b_r;
      rb = make_float4(0, 0, 0, 0);
      if (r < r_end) {
        const int br = d.bR[r];
        if (b_ok[3]) {
          rb = ld4(Bp + b_off[0] + br);
        } else {
          float v[4] = {0, 0, 0, 0};
#pragma unroll
          for (int i = 0; i < 4; ++i)
            if (b_ok[i]) v[i] = Bp[b_off[i] + br];
          rb = make_float4(v[0], v[1], v[2], v[3]);
        }
      }
    }
  };

  auto store_tiles = [&]() {
    if (a_rvec) {
      As[a_r + 0][a_m] = ra.x; As[a_r + 1][a_m] = ra.y; As[a_r + 2][a_m] = ra.z; As[a_r + 3][a_m] = ra.w;
    } else {
      *reinterpret_cast<float4*>(&As[a_r][a_m]) = ra;
    }
    if (b_rvec) {
      Bs[b_r + 0][b_n] = rb.x; Bs[b_r + 1][b_n] = rb.y; Bs[b_r + 2][b_n] = rb.z; Bs[b_r + 3][b_n] = rb.w;
    } else {
      *reinterpret_cast<float4*>(&Bs[b_r][b_n]) = rb;
      if (do_colsum) { csum[0] += rb.x; csum[1] += rb.y; csum[2] += rb.z; csum[3] += rb.w; }
    }
  };

  const int tx = tid & 15, ty = tid >> 4;
  Acc acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0;

  if (r_begin < r_end) load_tiles(r_begin);
  for (int rk = r_begin; rk < r_end; rk += BK) {
    store_tiles();
    __syncthreads();
    if (rk + BK < r_end) load_tiles(rk + BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if constexpr (EXT) acc[i][j] = fma((double)av[i], (double)bv[j], acc[i][j]);
          else acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
    }
    __syncthreads();
  }

  // ---- epilogue
  const int nb = n0 + tx * 4;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= d.M) continue;
    const int cm = d.cM[m];
    const int km = (d.flags & (EXT ? GG_EPI_MASK | GG_EPI_LRELU_GRAD : (TANH ? GG_EPI_MASK | GG_EPI_TANH_GRAD : GG_EPI_MASK))) ? (d.kM ? d.kM[m] : cm) : 0;
    float v[4];
    int co[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = nb + j;
      v[j] = (float)acc[i][j];
      co[j] = -1;
      if (n < d.N) {
        const int cn = d.cN[n];
        co[j] = cm + cn;
        if (d.flags & GG_EPI_BIAS_RELU) v[j] = fmaxf(v[j] + d.bias[n], 0.f);
        if (d.flags & GG_EPI_BIAS) v[j] += d.bias[n];
        if (d.flags & GG_EPI_BIAS_LRELU) {
          v[j] += d.bias[n];
          v[j] = v[j] > 0.f ? v[j] : d.alpha * v[j];
        }
        if (d.flags & GG_EPI_MASK) {
          const int kn = d.kN ? d.kN[n] : cn;
          v[j] = d.mask[km + kn] > 0.f ? v[j] : 0.f;
        }
        if (EXT && (d.flags & GG_EPI_LRELU_GRAD)) {
          const float a = d.mask[km + (d.kN ? d.kN[n] : cn)];
          v[j] *= a > 0.f ? 1.f : (a < 0.f ? d.alpha : 0.f);
        }
        if (TANH && (d.flags & GG_EPI_BIAS_TANH)) v[j] = tanhf(v[j] + d.bias[n]);
        if (TANH && (d.flags & GG_EPI_TANH_GRAD)) {
          const float y = d.mask[km + (d.kN ? d.kN[n] : cn)];
          v[j] *= 1.f - y * y;
        }
        if (d.flags & GG_EPI_SCALE) v[j] *= d.alpha;
      }
    }
    if (d.C_hi) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (co[j] >= 0) {
          const __nv_bfloat16 hh = __float2bfloat16_rn(v[j]);
          d.C_hi[co[j]] = __bfloat16_as_ushort(hh);
          d.C_lo[co[j]] = __bfloat16_as_ushort(__float2bfloat16_rn(v[j] - __bfloat162float(hh)));
        }
    }
    if (d.flags & GG_EPI_ATOMIC) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (co[j] >= 0) {
          if constexpr (EXT) atomicAdd(reinterpret_cast<double*>(d.C) + co[j], acc[i][j]);
          else atomicAdd(d.C + co[j], v[j]);
        }
    } else if (co[3] >= 0 && co[1] == co[0] + 1 && co[2] == co[0] + 2 && co[3] == co[0] + 3 && (co[0] & 3) == 0) {
      *reinterpret_cast<float4*>(d.C + co[0]) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (co[j] >= 0) d.C[co[j]] = v[j];
    }
  }
  if (do_colsum) {   // block-uniform branch
    atomicAdd(&cs[b_n + 0], csum[0]); atomicAdd(&cs[b_n + 1], csum[1]);
    atomicAdd(&cs[b_n + 2], csum[2]); atomicAdd(&cs[b_n + 3], csum[3]);
    __syncthreads();
    if (tid < BN && n0 + tid < d.N) {
      if constexpr (EXT) atomicAdd(reinterpret_cast<double*>(d.colsum) + n0 + tid, cs[tid]);
      else atomicAdd(d.colsum + n0 + tid, cs[tid]);
    }
  }
}

template <bool EXT>
__global__ void __launch_bounds__(256) gg_simt_kernel(const GemmDesc* __restrict__ descs, int ndesc) {
  gg_simt_body<EXT, false>(descs, ndesc);
}

__global__ void __launch_bounds__(256) gg_simt_tanh_kernel(const GemmDesc* __restrict__ descs, int ndesc) {
  gg_simt_body<false, true>(descs, ndesc);
}
}  // namespace

void gg_simt_launch(const GemmDesc* dev_descs, int ndesc, int total_tiles, cudaStream_t s) {
  if (total_tiles <= 0) return;
  launch_pdl(gg_simt_kernel<false>, dim3(total_tiles), dim3(256), 0, s, pdl_enabled(), dev_descs, ndesc);
}

void gg_simt_launch_ext(const GemmDesc* dev_descs, int ndesc, int total_tiles, cudaStream_t s) {
  if (total_tiles <= 0) return;
  gg_simt_kernel<true><<<total_tiles, 256, 0, s>>>(dev_descs, ndesc);
}

void gg_simt_launch_tanh(const GemmDesc* dev_descs, int ndesc, int total_tiles, cudaStream_t s) {
  if (total_tiles <= 0) return;
  gg_simt_tanh_kernel<<<total_tiles, 256, 0, s>>>(dev_descs, ndesc);
}

}  // namespace b2g
