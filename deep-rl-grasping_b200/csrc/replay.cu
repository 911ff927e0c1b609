// Replay rows: compaction of caller observations into compact rows, the frame pool's writes (frame_check / frame_commit), and
// the minibatch gather fused with VecNormalize and the policy's /255 input scaling.
//
// Row layout.  MLP policy: a row is the observation vector.  CNN policy: a row is COMPACT, Ec = H*W*Ci + 4 floats -- the
// image planes [H][W][Ci] (NHWC), then the one value of the constant actuator plane the network reads (pixel [0,0] of the last
// channel, custom_obs_policy.py:28-32; zero for the plain nature_cnn, whose rows hold all Ci planes of the observation), then
// 3 zero pads.  Callers pass full [H][W][Ci+1] (plain nature_cnn: [H][W][Ci]) observations; compact_kernel
// writes them into replay_add's staging, the explicit batch and policy inference's staging.  Replay frames hold such rows,
// optionally with 8-bit image channels (FrameFmt, common.cuh); the gathers decode them into the same fp32 values.
//
// gather_kernel restates [SB2] ReplayBuffer.sample(batch_size, env=vec_normalize) -> VecNormalize.normalize_obs /
// normalize_reward (configured at sb_helper.py:118-119: clip_obs=10, clip_reward=10, eps=1e-8; float64 arithmetic like numpy,
// cast to fp32 by the feed_dict) and observation_input(scale=True) ((x-0)/255 for the Box(0,255) of robot.py:224-228).
// HBM-bound: one coalesced pass over 2*B rows; no intermediate copies.  It serves the round-1 engines and policy inference;
// engine v2 reads the same rows with gather2_kernel (engine_v2.cu).
#include <cuda_bf16.h>

#include "common.cuh"

namespace b2g {
namespace {

// full observation [HW][Cfull] -> compact row {image planes [HW][Ci] | value at pixel [0,0] of plane Ci, or 0 | 3 pad}
__global__ void __launch_bounds__(256) compact_kernel(const float* __restrict__ src, float* __restrict__ dst, long long first_row, long long wrap,
                                                       int HW, int Ci, int Cfull, int Ec) {
  const float* s = src + (size_t)blockIdx.x * HW * Cfull;
  float* d = dst + (size_t)((first_row + blockIdx.x) % wrap) * Ec;
  for (int e = threadIdx.x; e < HW * Ci; e += blockDim.x) {
    const int pix = e / Ci, c = e - pix * Ci;
    d[e] = s[(size_t)pix * Cfull + c];
  }
  if (threadIdx.x < 4) d[HW * Ci + threadIdx.x] = threadIdx.x == 0 && Cfull > Ci ? s[Ci] : 0.f;
}

// float64 VecNormalize of the 4 row elements [e, e + 4) (e % 4 == 0): clip((x - mean) * istd, +-clip_obs)
__device__ __forceinline__ void load_norm4(const unsigned char* __restrict__ src, const GatherArgs& g, int npx, int e, bool norm_obs,
                                           double clip_obs, float y[4]) {
  const float4 v = frame_load4(src, g.fmt, npx, g.Cimg, e);
  y[0] = v.x; y[1] = v.y; y[2] = v.z; y[3] = v.w;
  if (norm_obs) {
    const double2 m0 = *reinterpret_cast<const double2*>(g.mean + e), m1 = *reinterpret_cast<const double2*>(g.mean + e + 2);
    const double2 s0 = *reinterpret_cast<const double2*>(g.var + e), s1 = *reinterpret_cast<const double2*>(g.var + e + 2);
    const double mm[4] = {m0.x, m0.y, m1.x, m1.y}, ss[4] = {s0.x, s0.y, s1.x, s1.y};   // ss = 1/sqrt(var+eps)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double d = ((double)y[j] - mm[j]) * ss[j];
      d = fmin(fmax(d, -clip_obs), clip_obs);
      y[j] = (float)d;
    }
  }
}

__global__ void __launch_bounds__(256) gather_kernel(GatherArgs g) {
  const int b = blockIdx.y;
  const int which = blockIdx.z;               // 0 = obs, 1 = next_obs
  const bool cnn = g.H > 0;
  const int npx = g.H * g.W * g.Cimg;         // CNN: image elements of a row (index of the actuator value)
  const int E = cnn ? npx + 4 : g.W;
  long long slot = b;
  if (g.indices) slot = g.indices[b];
  else if (g.rng_counters) {
    slot = philox_slot(g.seed, (unsigned long long)g.rng_counters[4], b, (unsigned long long)g.rng_counters[5]);
    if (g.ring_cap > 0) slot = ring_slot(g.rng_counters[6], (int)slot, g.ring_cap);
    if (g.indices_out && which == 0 && blockIdx.x == 0 && threadIdx.x == 0) g.indices_out[b] = (int)slot;
  }
  const unsigned char* __restrict__ fsrc =
      g.obs_frame ? g.frames + (size_t)(which ? g.next_frame : g.obs_frame)[slot] * g.frame_bytes
                  : reinterpret_cast<const unsigned char*>((which ? g.next_obs : g.obs) + (size_t)slot * E);
  const float* __restrict__ src = reinterpret_cast<const float*>(fsrc);   // MLP rows: always fp32
  const double ret_istd = g.normc[0], clip_obs = g.normc[1], clip_rew = g.normc[2];
  const bool norm_obs = g.normc[3] != 0.0, norm_rew = g.normc[4] != 0.0;
  const float inv_scale_denom = g.scale;
  if (cnn) {
    // the image block is exactly the NHWC input x with Ci channels: 4-element group e4 of the row is group e4 of the sample's x
    // (and of its BF16 planes).  b2g_sac_create requires (W * Ci) % 4 == 0, so npx and Ec are multiples of 4 and every 128-bit
    // access here is aligned.
    const size_t o = (size_t)b * npx;
    float* __restrict__ xdst = (which ? g.x_next : g.x_obs) + o;
    uint16_t* __restrict__ xhi = which ? g.x_next_hi : g.x_obs_hi;
    uint16_t* __restrict__ xlo = which ? g.x_next_lo : g.x_obs_lo;
    for (int e4 = blockIdx.x * blockDim.x + threadIdx.x; e4 < (npx >> 2); e4 += gridDim.x * blockDim.x) {
      float y[4];
      load_norm4(fsrc, g, npx, 4 * e4, norm_obs, clip_obs, y);
#pragma unroll
      for (int j = 0; j < 4; ++j) y[j] = y[j] / inv_scale_denom;
      *reinterpret_cast<float4*>(xdst + 4 * e4) = make_float4(y[0], y[1], y[2], y[3]);
      if (xhi) {
        uint16_t hi[4], lo[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const __nv_bfloat16 h = __float2bfloat16_rn(y[j]);
          hi[j] = __bfloat16_as_ushort(h);
          lo[j] = __bfloat16_as_ushort(__float2bfloat16_rn(y[j] - __bfloat162float(h)));
        }
        *reinterpret_cast<uint2*>(xhi + o + 4 * e4) = make_uint2((uint32_t)hi[0] | ((uint32_t)hi[1] << 16), (uint32_t)hi[2] | ((uint32_t)hi[3] << 16));
        *reinterpret_cast<uint2*>(xlo + o + 4 * e4) = make_uint2((uint32_t)lo[0] | ((uint32_t)lo[1] << 16), (uint32_t)lo[2] | ((uint32_t)lo[3] << 16));
      }
    }
    if (g.feat_col >= 0 && blockIdx.x == 0 && threadIdx.x == 0) {      // the actuator value -> the direct-feature column
      float y = frame_elem(fsrc, g.fmt, npx, g.Cimg, npx);
      if (norm_obs) y = (float)fmin(fmax(((double)y - g.mean[npx]) * g.var[npx], -clip_obs), clip_obs);
      y = y / inv_scale_denom;
      if (which) g.F_t[(size_t)b * g.FS + g.feat_col] = y;
      else { g.F_pi[(size_t)b * g.FS + g.feat_col] = y; g.F_v[(size_t)b * g.FS + g.feat_col] = y; }
    }
  } else {
    // 4 consecutive elements per thread (128-bit loads) when the observation length allows it
    const int E4 = (E & 3) == 0 ? E >> 2 : 0;
    for (int e4 = blockIdx.x * blockDim.x + threadIdx.x; e4 < E4; e4 += gridDim.x * blockDim.x) {
      float y[4];
      load_norm4(fsrc, g, 0, 4 * e4, norm_obs, clip_obs, y);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int e = 4 * e4 + j;
        const float yy = y[j] / inv_scale_denom;
        if (which) g.F_t[(size_t)b * g.FS + e] = yy;
        else { g.F_pi[(size_t)b * g.FS + e] = yy; g.F_v[(size_t)b * g.FS + e] = yy; }
      }
    }
    if (E4 == 0) {   // generic scalar path
      for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < E; e += gridDim.x * blockDim.x) {
        float y = src[e];
        if (norm_obs) {
          double d = ((double)y - g.mean[e]) * g.var[e];
          d = fmin(fmax(d, -clip_obs), clip_obs);
          y = (float)d;
        }
        y = y / g.scale;
        if (which) g.F_t[(size_t)b * g.FS + e] = y;
        else { g.F_pi[(size_t)b * g.FS + e] = y; g.F_v[(size_t)b * g.FS + e] = y; }
      }
    }
  }
  if (which == 0 && blockIdx.x == 0 && g.act) {
    const int feat_dim = cnn ? g.act_col : g.W;
    if (threadIdx.x < g.n_act) g.F_v[(size_t)b * g.FS + feat_dim + threadIdx.x] = g.act[slot * g.n_act + threadIdx.x];
    if (threadIdx.x == 32) {
      float r = g.rew[slot];
      if (norm_rew) {
        double d = (double)r * ret_istd;
        d = fmin(fmax(d, -clip_rew), clip_rew);
        r = (float)d;
      }
      g.rew_out[b] = r;
      g.done_out[b] = g.done[slot];
    }
  }
}
__device__ __forceinline__ bool u8_channel(const FrameIo& io, int e) {
  return io.fmt.n8 > 0 && e < io.npx && io.fmt.ch[e % io.Ci] >= 0;
}

// one CTA per row (see frame_check_launch)
__global__ void __launch_bounds__(256) frame_check_kernel(FrameIo io, const int* __restrict__ prev, int* __restrict__ flags) {
  __shared__ int s_neq, s_bad;
  const int i = blockIdx.x;
  if (threadIdx.x == 0) { s_neq = 0; s_bad = 0; }
  __syncthreads();
  const float* o = io.c_obs + (size_t)i * io.Ec;
  const float* nx = io.c_next + (size_t)i * io.Ec;
  const int p = prev[i];
  const unsigned char* f = p >= 0 ? io.frames + (size_t)p * io.frame_bytes : nullptr;
  int neq = 0, bad = 0;
  for (int e = threadIdx.x; e < io.Ec; e += blockDim.x) {
    const float v = o[e];
    if (f && __float_as_uint(frame_elem(f, io.fmt, io.npx, io.Ci, e)) != __float_as_uint(v)) neq = 1;
    if (u8_channel(io, e)) {
      // -0.0 would come back as +0.0: refused with the fractions, negatives, values > 255 and NaNs
      const float w = nx[e];
      if (!(v >= 0.f && v <= 255.f && v == rintf(v) && !signbit(v))) bad = 1;
      if (!(w >= 0.f && w <= 255.f && w == rintf(w) && !signbit(w))) bad = 1;
    }
  }
  if (neq) atomicOr(&s_neq, 1);
  if (bad) atomicOr(&s_bad, 1);
  __syncthreads();
  if (threadIdx.x == 0) flags[i] = (f && !s_neq ? 1 : 0) | (s_bad ? 2 : 0);
}

// grid (m, 2): y = 0 writes the obs row (when it takes a new frame) and the transition's frame indices, y = 1 the next_obs row.
// plan == nullptr: every row takes two new frames, ids fid0 + 2i and fid0 + 2i + 1.
__global__ void __launch_bounds__(256) frame_commit_kernel(FrameIo io, const int* __restrict__ plan, long long fid0, long long fcap,
                                                           int m, int* __restrict__ r_ofr, int* __restrict__ r_nfr, long long first,
                                                           long long cap) {
  const int i = blockIdx.x, which = blockIdx.y;
  const int of = plan ? plan[i] : (int)((fid0 + 2 * i) % fcap);
  const int nf = plan ? plan[2 * m + i] : (int)((fid0 + 2 * i + 1) % fcap);
  if (which == 0 && threadIdx.x == 0) {
    const long long slot = (first + i) % cap;
    r_ofr[slot] = of;
    r_nfr[slot] = nf;
  }
  if (which == 0 && plan && !plan[m + i]) return;
  const float* src = (which ? io.c_next : io.c_obs) + (size_t)i * io.Ec;
  unsigned char* f = io.frames + (size_t)(which ? nf : of) * io.frame_bytes;
  const FrameFmt& fm = io.fmt;
  for (int e = threadIdx.x; e < io.Ec; e += blockDim.x) {
    const float v = src[e];
    if (e >= io.npx) { reinterpret_cast<float*>(f + fm.tail)[e - io.npx] = v; continue; }
    if (fm.n8 == 0) { reinterpret_cast<float*>(f)[e] = v; continue; }
    const int pix = e / io.Ci, k = fm.ch[e - pix * io.Ci];
    if (k >= 0) f[pix * fm.n8 + k] = (unsigned char)v;
    else reinterpret_cast<float*>(f + fm.f32_off)[pix * fm.n32 - 1 - k] = v;
  }
}
}  // namespace

void frame_check_launch(const FrameIo& io, const int* prev, int* flags, int m, cudaStream_t s) {
  if (m > 0) frame_check_kernel<<<m, 256, 0, s>>>(io, prev, flags);
}

void frame_commit_launch(const FrameIo& io, const int* plan, long long fid0, long long fcap, int m, int* r_ofr, int* r_nfr,
                         long long first, long long cap, cudaStream_t s) {
  if (m > 0) frame_commit_kernel<<<dim3(m, 2), 256, 0, s>>>(io, plan, fid0, fcap, m, r_ofr, r_nfr, first, cap);
}

void compact_rows(const float* src_full, float* dst, long long first_row, long long wrap, int n, int HW, int Ci, int Cfull,
                  cudaStream_t s) {
  if (n > 0) compact_kernel<<<n, 256, 0, s>>>(src_full, dst, first_row, wrap, HW, Ci, Cfull, HW * Ci + 4);
}

void gather_launch(const GatherArgs& a, cudaStream_t s) {
  const int E = a.H > 0 ? a.H * a.W * a.Cimg + 4 : a.W;
  int gx = (E / 4 + 255) / 256;      // one 128-bit group per thread
  if (gx < 1) gx = 1;
  if (gx > 4) gx = 4;
  dim3 grid(gx, a.B, a.next_obs || a.next_frame ? 2 : 1);
  gather_kernel<<<grid, 256, 0, s>>>(a);
}

}  // namespace b2g
