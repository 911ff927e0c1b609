// Fused head "tail": everything between the fc0 contractions and their gradients, four warps per
// sample (coalesced HBM/L2 reads, warp-shuffle reductions, no tensor cores: these are 64-wide
// latency-bound layers).
//
// Restates [SB2] sac/policies.py make_actor / make_critics after the first dense layer, and
// [SB2] sac/sac.py setup_model's loss block (SURVEY.md Appendix A):
//   actor  : a0=relu(z0+b0) -> fc1 -> mu, log_std(clip) -> u=mu+eps*std -> pi=tanh(u), logp
//   critics: vf, qf1, qf2 at the replay action; qf1, qf2 at pi (fc0 reused: z0(pi)=z0(a)+(pi-a)K0[act rows])
//   target : vf_target(next)
//   losses : qf1/qf2/value/policy/ent_coef + their backward seeds, back-propagated to dz0 per head
// Outputs feed the gather-GEMM engine (fc0 wgrad/dgrad); the tiny output-layer gradients are
// reduced in shared memory and added to the gradient arena here.
#include <math.h>

#include <cuda_bf16.h>

#include "common.cuh"

namespace b2g {
namespace {
constexpr int H = 64, LD = 65, WARPS = 8, AMAX = 8;
constexpr float EPSF = 1e-6f, LS_MAX = 2.0f, LS_MIN = -20.0f;

struct V2 { float lo, hi; };

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ V2 relu2(V2 a) { return V2{fmaxf(a.lo, 0.f), fmaxf(a.hi, 0.f)}; }

// out[j] = bias[j] + sum_i a[i] * W[i][j]
__device__ __forceinline__ V2 fwd64(const float* __restrict__ Ws, const float* __restrict__ bias, V2 a, int lane) {
  V2 o{bias[lane], bias[lane + 32]};
#pragma unroll 8
  for (int i = 0; i < 32; ++i) {
    const float ai = __shfl_sync(0xffffffffu, a.lo, i);
    o.lo = fmaf(ai, Ws[i * LD + lane], o.lo);
    o.hi = fmaf(ai, Ws[i * LD + lane + 32], o.hi);
  }
#pragma unroll 8
  for (int i = 0; i < 32; ++i) {
    const float ai = __shfl_sync(0xffffffffu, a.hi, i);
    o.lo = fmaf(ai, Ws[(i + 32) * LD + lane], o.lo);
    o.hi = fmaf(ai, Ws[(i + 32) * LD + lane + 32], o.hi);
  }
  return o;
}
// out[i] = sum_j dz[j] * W[i][j]
__device__ __forceinline__ V2 bwd64(const float* __restrict__ Ws, V2 dz, int lane) {
  V2 o{0.f, 0.f};
#pragma unroll 8
  for (int j = 0; j < 32; ++j) {
    const float dj = __shfl_sync(0xffffffffu, dz.lo, j);
    o.lo = fmaf(dj, Ws[lane * LD + j], o.lo);
    o.hi = fmaf(dj, Ws[(lane + 32) * LD + j], o.hi);
  }
#pragma unroll 8
  for (int j = 0; j < 32; ++j) {
    const float dj = __shfl_sync(0xffffffffu, dz.hi, j);
    o.lo = fmaf(dj, Ws[lane * LD + j + 32], o.lo);
    o.hi = fmaf(dj, Ws[(lane + 32) * LD + j + 32], o.hi);
  }
  return o;
}
// N independent 64x64 mat-vecs advanced in lock step: same arithmetic (and order) per mat-vec as fwd64, but the N
// dependent FMA chains and their shuffles / shared loads interleave, so the warp's duration is the length of one
// dependency chain, not N of them.
template <int N>
__device__ __forceinline__ void fwd64xN(const float* const (&Ws)[N], const float* const (&bias)[N], const V2 (&a)[N], V2 (&o)[N], int lane) {
#pragma unroll
  for (int k = 0; k < N; ++k) o[k] = V2{bias[k][lane], bias[k][lane + 32]};
#pragma unroll 4
  for (int i = 0; i < 32; ++i) {
#pragma unroll
    for (int k = 0; k < N; ++k) {
      const float ai = __shfl_sync(0xffffffffu, a[k].lo, i);
      o[k].lo = fmaf(ai, Ws[k][i * LD + lane], o[k].lo);
      o[k].hi = fmaf(ai, Ws[k][i * LD + lane + 32], o[k].hi);
    }
  }
#pragma unroll 4
  for (int i = 0; i < 32; ++i) {
#pragma unroll
    for (int k = 0; k < N; ++k) {
      const float ai = __shfl_sync(0xffffffffu, a[k].hi, i);
      o[k].lo = fmaf(ai, Ws[k][(i + 32) * LD + lane], o[k].lo);
      o[k].hi = fmaf(ai, Ws[k][(i + 32) * LD + lane + 32], o[k].hi);
    }
  }
}
__device__ __forceinline__ V2 ld2(const float* p, int lane) { return V2{p[lane], p[lane + 32]}; }
__device__ __forceinline__ void st2(float* p, int lane, V2 v) { p[lane] = v.lo; p[lane + 32] = v.hi; }
// BF16 hi / lo planes of a 64-wide row (x = hi + lo to ~2^-17)
__device__ __forceinline__ void st2_planes(uint16_t* hi, uint16_t* lo, int lane, V2 v) {
  const __nv_bfloat16 h0 = __float2bfloat16_rn(v.lo), h1 = __float2bfloat16_rn(v.hi);
  hi[lane] = __bfloat16_as_ushort(h0); hi[lane + 32] = __bfloat16_as_ushort(h1);
  lo[lane] = __bfloat16_as_ushort(__float2bfloat16_rn(v.lo - __bfloat162float(h0)));
  lo[lane + 32] = __bfloat16_as_ushort(__float2bfloat16_rn(v.hi - __bfloat162float(h1)));
}
// scalar head output: sum_i a[i]*ko[i] + bo
__device__ __forceinline__ float out1(const float* __restrict__ ko, const float* __restrict__ bo, V2 a, int lane) {
  return warp_sum(a.lo * ko[lane] + a.hi * ko[lane + 32]) + bo[0];
}

enum { S_PI = 0, S_VF, S_Q1, S_Q2, S_VT, S_NW };

// ================================================================================================
// tail4: the per-sample work is split over FOUR warps (actor | vf + target vf | qf1 | qf2) that exchange a
// handful of scalars through shared memory and three named barriers.  A warp's duration is its dependency
// chain: with one warp per sample it is 12 serial 64x64 mat-vecs, here 4 (actor fc1 -> qf1-at-pi fc1 ->
// qf1-at-pi fc1^T -> actor fc1^T), and 128 CTAs instead of 32 occupy the GPU.
// ================================================================================================
__device__ __forceinline__ void bar_group(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

__global__ void __launch_bounds__(WARPS * 32) tail4_kernel(TailArgs t) {
  extern __shared__ float smem[];
  float* Wk1 = smem;
  float* acc = Wk1 + S_NW * H * LD;
  const int A = t.A;
  const int n_acc = 2 * H * A + 2 * A + 3 * (H + 1);
  float* red = acc + n_acc;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  pdl_trigger();
  pdl_wait();
  const float* k1s[S_NW] = {t.pi.k1, t.vf.k1, t.q1.k1, t.q2.k1, t.vt.k1};
  for (int w = 0; w < S_NW; ++w)
    for (int i = tid; i < H * H; i += blockDim.x) {
      const uint32_t dst = (uint32_t)__cvta_generic_to_shared(&Wk1[w * H * LD + (i >> 6) * LD + (i & 63)]);
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(k1s[w] + i) : "memory");
    }
  float* sp = red + ((MET_COUNT + 1 + 3) & ~3);
  auto stage = [&](float* dst, const float* src, int n) {
    for (int i = tid; i < n; i += blockDim.x) {
      const uint32_t d32 = (uint32_t)__cvta_generic_to_shared(dst + i);
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d32), "l"(src + i) : "memory");
    }
  };
  const HeadW* hw[S_NW] = {&t.pi, &t.vf, &t.q1, &t.q2, &t.vt};
  float* s_b0[S_NW]; float* s_b1[S_NW];
  for (int w = 0; w < S_NW; ++w) {
    s_b0[w] = sp + w * 2 * H; s_b1[w] = s_b0[w] + H;
    stage(s_b0[w], hw[w]->b0, H); stage(s_b1[w], hw[w]->b1, H);
  }
  float* s_pi_ko = sp + S_NW * 2 * H;
  float* s_ksig = s_pi_ko + H * A;
  float* s_pi_bo = s_ksig + H * A;
  float* s_bsig = s_pi_bo + A;
  float* s_vko[4];
  s_vko[0] = s_bsig + A;
  for (int w = 1; w < 4; ++w) s_vko[w] = s_vko[w - 1] + H + 1;
  float* s_q1act = s_vko[3] + H + 1;
  float* s_q2act = s_q1act + A * H;
  float* scratch = s_q2act + A * H;               // 2 sample groups x 32 floats
  stage(s_pi_ko, t.pi.ko, H * A); stage(s_ksig, t.ksig, H * A); stage(s_pi_bo, t.pi.bo, A); stage(s_bsig, t.bsig, A);
  {
    const HeadW* vh[4] = {&t.vf, &t.q1, &t.q2, &t.vt};
    for (int w = 0; w < 4; ++w) { stage(s_vko[w], vh[w]->ko, H); stage(s_vko[w] + H, vh[w]->bo, 1); }
  }
  stage(s_q1act, t.q1.k0 + (size_t)t.feat_dim * H, A * H);
  stage(s_q2act, t.q2.k0 + (size_t)t.feat_dim * H, A * H);
  for (int i = tid; i < n_acc + MET_COUNT + 1; i += blockDim.x) acc[i] = 0.f;
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();

  float* a_kmu = acc;
  float* a_ksig = a_kmu + H * A;
  float* a_bmu = a_ksig + H * A;
  float* a_bsig = a_bmu + A;
  float* a_vf = a_bsig + A;
  float* a_q1 = a_vf + H + 1;
  float* a_q2 = a_q1 + H + 1;
  const float invB = 1.0f / (float)t.grad_scale_B;
  const float log_alpha = t.log_alpha[0];
  const float alpha = expf(log_alpha);
  const int sg = warp >> 2, role = warp & 3, barid = 1 + sg;
  float* sc = scratch + sg * 32;          // [0..7] pi, [8] logp, [9] q1p, [10] q2p, [11] v_targ, [16..23] dpi

  for (int b = blockIdx.x * 2 + sg; b < t.B; b += gridDim.x * 2) {
    if (role == 0) {
      // ------------------------------------------------------------------ actor
      const V2 zpi = ld2(t.z0_pi + b * H, lane);
      float eps_r[AMAX];
#pragma unroll
      for (int a = 0; a < AMAX; ++a) eps_r[a] = a < A ? t.eps[b * A + a] : 0.f;
      const V2 a0_pi = relu2(V2{zpi.lo + s_b0[S_PI][lane], zpi.hi + s_b0[S_PI][lane + 32]});
      st2(t.a0_pi + b * H, lane, a0_pi);
      const V2 g = relu2(fwd64(Wk1 + S_PI * H * LD, s_b1[S_PI], a0_pi, lane));
      float mu[AMAX], ls_raw[AMAX], ls[AMAX], sd[AMAX], pi[AMAX], tt[AMAX];
      float logp = 0.f, ent = 0.f;
#pragma unroll
      for (int a = 0; a < AMAX; ++a) {
        if (a < A) {
          mu[a] = warp_sum(g.lo * s_pi_ko[lane * A + a] + g.hi * s_pi_ko[(lane + 32) * A + a]) + s_pi_bo[a];
          ls_raw[a] = warp_sum(g.lo * s_ksig[lane * A + a] + g.hi * s_ksig[(lane + 32) * A + a]) + s_bsig[a];
          ls[a] = fminf(fmaxf(ls_raw[a], LS_MIN), LS_MAX);
          sd[a] = expf(ls[a]);
          const float u = mu[a] + eps_r[a] * sd[a];
          tt[a] = (u - mu[a]) / (sd[a] + EPSF);
          pi[a] = tanhf(u);
          logp += -0.5f * (tt[a] * tt[a] + 2.f * ls[a] + 1.8378770664093453f) - logf(1.f - pi[a] * pi[a] + EPSF);
          ent += ls[a] + 1.4189385332046727f;
          if (lane == a) sc[a] = pi[a];
        }
      }
      if (lane == 0) sc[8] = logp;
      bar_group(barid);                                    // A: pi, logp published
      bar_group(barid);                                    // B: q1p, q2p, v_targ published
      const float q1p = sc[9];
      if (lane == 0) {
        atomicAdd(&red[MET_POLICY_LOSS], (alpha * logp - q1p) * invB);
        atomicAdd(&red[MET_ENT_COEF_LOSS], -log_alpha * (logp + t.target_entropy) * invB);
        atomicAdd(&red[MET_ENTROPY], ent * invB);
        atomicAdd(&red[MET_MEAN_LOGP], logp * invB);
        atomicAdd(&red[MET_COUNT], -(logp + t.target_entropy) * invB);
        if (t.per_sample) t.per_sample[3 * t.B + b] = logp;
      }
      if (t.pi_out && lane < A) {
        float pv = 0.f;
#pragma unroll
        for (int a = 0; a < AMAX; ++a) if (a == lane) pv = pi[a];
        t.pi_out[b * A + lane] = pv;
      }
      bar_group(barid);                                    // C: dpi published
      float dmu[AMAX], dls[AMAX];
      V2 dg{0.f, 0.f};
#pragma unroll
      for (int a = 0; a < AMAX; ++a) {
        if (a < A) {
          const float dpi = sc[16 + a];
          const float one_m = 1.f - pi[a] * pi[a];
          const float du = (alpha * invB) * 2.f * pi[a] * one_m / (one_m + EPSF) + dpi * one_m;
          dmu[a] = du;
          const float spe = sd[a] + EPSF;
          float d = du * eps_r[a] * sd[a] + (alpha * invB) * (-tt[a] * eps_r[a] * sd[a] * EPSF / (spe * spe) - 1.f);
          dls[a] = (ls_raw[a] >= LS_MIN && ls_raw[a] <= LS_MAX) ? d : 0.f;
          atomicAdd(&a_kmu[lane * A + a], g.lo * dmu[a]);
          atomicAdd(&a_kmu[(lane + 32) * A + a], g.hi * dmu[a]);
          atomicAdd(&a_ksig[lane * A + a], g.lo * dls[a]);
          atomicAdd(&a_ksig[(lane + 32) * A + a], g.hi * dls[a]);
          if (lane == 0) { atomicAdd(&a_bmu[a], dmu[a]); atomicAdd(&a_bsig[a], dls[a]); }
          dg.lo += dmu[a] * s_pi_ko[lane * A + a] + dls[a] * s_ksig[lane * A + a];
          dg.hi += dmu[a] * s_pi_ko[(lane + 32) * A + a] + dls[a] * s_ksig[(lane + 32) * A + a];
        }
      }
      const V2 dz1{g.lo > 0.f ? dg.lo : 0.f, g.hi > 0.f ? dg.hi : 0.f};
      st2(t.dz1_pi + b * H, lane, dz1);
      const V2 da0 = bwd64(Wk1 + S_PI * H * LD, dz1, lane);
      const V2 dz0{a0_pi.lo > 0.f ? da0.lo : 0.f, a0_pi.hi > 0.f ? da0.hi : 0.f};
      st2(t.dz0_pi + b * H, lane, dz0);
      if (t.dz0_pi_p[0]) st2_planes(t.dz0_pi_p[0] + (size_t)b * H, t.dz0_pi_p[1] + (size_t)b * H, lane, dz0);
    } else if (role == 1) {
      // ------------------------------------------------------------------ vf + target vf
      const V2 zvf = ld2(t.z0_vf + (size_t)b * t.z0v_ld, lane), zvt = ld2(t.z0_vt + b * H, lane);
      const V2 a0_vf = relu2(V2{zvf.lo + s_b0[S_VF][lane], zvf.hi + s_b0[S_VF][lane + 32]});
      const V2 a0_vt = relu2(V2{zvt.lo + s_b0[S_VT][lane], zvt.hi + s_b0[S_VT][lane + 32]});
      V2 a1_vf, a1_vt;
      {
        const float* const Wn[2] = {Wk1 + S_VF * H * LD, Wk1 + S_VT * H * LD};
        const float* const bn[2] = {s_b1[S_VF], s_b1[S_VT]};
        const V2 an[2] = {a0_vf, a0_vt};
        V2 on[2];
        fwd64xN<2>(Wn, bn, an, on, lane);
        a1_vf = relu2(on[0]); a1_vt = relu2(on[1]);
      }
      const float v = out1(s_vko[0], s_vko[0] + H, a1_vf, lane);
      const float v_targ = out1(s_vko[3], s_vko[3] + H, a1_vt, lane);
      if (lane == 0) sc[11] = v_targ;
      bar_group(barid);                                    // A
      bar_group(barid);                                    // B
      const float v_backup = fminf(sc[9], sc[10]) - alpha * sc[8];
      const float ev = v - v_backup;
      if (lane == 0) {
        atomicAdd(&red[MET_VALUE_LOSS], 0.5f * ev * ev * invB);
        atomicAdd(&red[MET_MEAN_V], v * invB);
        if (t.per_sample) { t.per_sample[2 * t.B + b] = v; t.per_sample[4 * t.B + b] = v_targ; }
      }
      st2(t.a0_vf + b * H, lane, a0_vf);
      const float dout = ev * invB;
      atomicAdd(&a_vf[lane], a1_vf.lo * dout);
      atomicAdd(&a_vf[lane + 32], a1_vf.hi * dout);
      if (lane == 0) atomicAdd(&a_vf[H], dout);
      const V2 dz1{a1_vf.lo > 0.f ? dout * s_vko[0][lane] : 0.f, a1_vf.hi > 0.f ? dout * s_vko[0][lane + 32] : 0.f};
      st2(t.dz1_vf + b * H, lane, dz1);
      const V2 da = bwd64(Wk1 + S_VF * H * LD, dz1, lane);
      const V2 dz0{a0_vf.lo > 0.f ? da.lo : 0.f, a0_vf.hi > 0.f ? da.hi : 0.f};
      st2(t.dz0_v3 + (size_t)b * 3 * H, lane, dz0);
      if (t.dz0_v3_p[0]) st2_planes(t.dz0_v3_p[0] + (size_t)b * 3 * H, t.dz0_v3_p[1] + (size_t)b * 3 * H, lane, dz0);
      bar_group(barid);                                    // C
    } else {
      // ------------------------------------------------------------------ qf1 (role 2) / qf2 (role 3)
      const bool isq1 = role == 2;
      const int SQ = isq1 ? S_Q1 : S_Q2;
      const float* z0p = isq1 ? t.z0_q1 : t.z0_q2;
      const float* sact = isq1 ? s_q1act : s_q2act;
      const float* sko = isq1 ? s_vko[1] : s_vko[2];
      float* aacc = isq1 ? a_q1 : a_q2;
      const V2 z0q = ld2(z0p + (size_t)b * t.z0v_ld, lane);
      const float rew_r = t.rew[b], done_r = t.done[b];
      float act_r[AMAX];
#pragma unroll
      for (int a = 0; a < AMAX; ++a) act_r[a] = a < A ? t.act[(size_t)b * t.act_stride + a] : 0.f;
      const V2 b0q = ld2(s_b0[SQ], lane);
      const V2 a0_q = relu2(V2{z0q.lo + b0q.lo, z0q.hi + b0q.hi});
      const V2 a1_q = relu2(fwd64(Wk1 + SQ * H * LD, s_b1[SQ], a0_q, lane));
      const float q = out1(sko, sko + H, a1_q, lane);
      bar_group(barid);                                    // A: pi available
      V2 z0qp = z0q;
#pragma unroll
      for (int a = 0; a < AMAX; ++a) {
        if (a < A) {
          const float dlt = sc[a] - act_r[a];
          const float* r1 = sact + a * H;
          z0qp.lo = fmaf(dlt, r1[lane], z0qp.lo); z0qp.hi = fmaf(dlt, r1[lane + 32], z0qp.hi);
        }
      }
      const V2 a0_qp = relu2(V2{z0qp.lo + b0q.lo, z0qp.hi + b0q.hi});
      const V2 a1_qp = relu2(fwd64(Wk1 + SQ * H * LD, s_b1[SQ], a0_qp, lane));
      const float qp = out1(sko, sko + H, a1_qp, lane);
      if (lane == 0) sc[isq1 ? 9 : 10] = qp;
      bar_group(barid);                                    // B
      if (isq1) {
        // d(-Q1(s, pi))/d pi first: the actor warp waits for it
        const float dout = -invB;
        const V2 dzp{a1_qp.lo > 0.f ? dout * sko[lane] : 0.f, a1_qp.hi > 0.f ? dout * sko[lane + 32] : 0.f};
        const V2 dap = bwd64(Wk1 + SQ * H * LD, dzp, lane);
        const V2 dz0p{a0_qp.lo > 0.f ? dap.lo : 0.f, a0_qp.hi > 0.f ? dap.hi : 0.f};
#pragma unroll
        for (int a = 0; a < AMAX; ++a) {
          if (a < A) {
            const float* r1 = sact + a * H;
            const float d = warp_sum(dz0p.lo * r1[lane] + dz0p.hi * r1[lane + 32]);
            if (lane == a) sc[16 + a] = d;
          }
        }
      }
      bar_group(barid);                                    // C
      const float q_backup = rew_r + (1.f - done_r) * t.gamma * sc[11];
      const float e = q - q_backup;
      if (lane == 0) {
        atomicAdd(&red[isq1 ? MET_QF1_LOSS : MET_QF2_LOSS], 0.5f * e * e * invB);
        atomicAdd(&red[isq1 ? MET_MEAN_Q1 : MET_MEAN_Q2], q * invB);
        if (t.per_sample) { t.per_sample[(isq1 ? 0 : 1) * t.B + b] = q; t.per_sample[(isq1 ? 5 : 6) * t.B + b] = qp; }
      }
      st2((isq1 ? t.a0_q1 : t.a0_q2) + b * H, lane, a0_q);
      const float dout = e * invB;
      atomicAdd(&aacc[lane], a1_q.lo * dout);
      atomicAdd(&aacc[lane + 32], a1_q.hi * dout);
      if (lane == 0) atomicAdd(&aacc[H], dout);
      const V2 dz1{a1_q.lo > 0.f ? dout * sko[lane] : 0.f, a1_q.hi > 0.f ? dout * sko[lane + 32] : 0.f};
      st2((isq1 ? t.dz1_q1 : t.dz1_q2) + b * H, lane, dz1);
      const V2 da = bwd64(Wk1 + SQ * H * LD, dz1, lane);
      const V2 dz0{a0_q.lo > 0.f ? da.lo : 0.f, a0_q.hi > 0.f ? da.hi : 0.f};
      const size_t o = (size_t)b * 3 * H + (isq1 ? H : 2 * H);
      st2(t.dz0_v3 + o, lane, dz0);
      if (t.dz0_v3_p[0]) st2_planes(t.dz0_v3_p[0] + o, t.dz0_v3_p[1] + o, lane, dz0);
    }
  }
  __syncthreads();
  for (int i = tid; i < H * A; i += blockDim.x) {
    atomicAdd(t.g_pi.ko + i, a_kmu[i]);
    atomicAdd(t.g_ksig + i, a_ksig[i]);
  }
  if (tid < A) { atomicAdd(t.g_pi.bo + tid, a_bmu[tid]); atomicAdd(t.g_bsig + tid, a_bsig[tid]); }
  if (tid < H) {
    atomicAdd(t.g_vf.ko + tid, a_vf[tid]); atomicAdd(t.g_q1.ko + tid, a_q1[tid]); atomicAdd(t.g_q2.ko + tid, a_q2[tid]);
  }
  if (tid == 0) {
    atomicAdd(t.g_vf.bo, a_vf[H]); atomicAdd(t.g_q1.bo, a_q1[H]); atomicAdd(t.g_q2.bo, a_q2[H]);
    atomicAdd(t.g_log_alpha, red[MET_COUNT]);
  }
  if (tid < MET_GN_PI) atomicAdd(t.metrics + tid, red[tid]);
}

// ---- policy inference ([SB2] SACPolicy.step: deterministic_policy = tanh(mu), policy = tanh(mu + eps*std))
__global__ void __launch_bounds__(WARPS * 32) act_kernel(TailArgs t, int n, int deterministic, float* act_out) {
  __shared__ float Wk1[H * LD];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < H * H; i += blockDim.x) {
    const uint32_t dst = (uint32_t)__cvta_generic_to_shared(&Wk1[(i >> 6) * LD + (i & 63)]);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(t.pi.k1 + i) : "memory");
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();
  const int A = t.A;
  for (int b = blockIdx.x * WARPS + warp; b < n; b += gridDim.x * WARPS) {
    const V2 a0 = relu2(V2{t.z0_pi[b * H + lane] + t.pi.b0[lane], t.z0_pi[b * H + lane + 32] + t.pi.b0[lane + 32]});
    const V2 g = relu2(fwd64(Wk1, t.pi.b1, a0, lane));
    for (int a = 0; a < A; ++a) {
      const float mu = warp_sum(g.lo * t.pi.ko[lane * A + a] + g.hi * t.pi.ko[(lane + 32) * A + a]) + t.pi.bo[a];
      float u = mu;
      if (!deterministic) {
        float ls = warp_sum(g.lo * t.ksig[lane * A + a] + g.hi * t.ksig[(lane + 32) * A + a]) + t.bsig[a];
        ls = fminf(fmaxf(ls, LS_MIN), LS_MAX);
        u = mu + t.eps[b * A + a] * expf(ls);
      }
      if (lane == 0) act_out[b * A + a] = tanhf(u);
    }
  }
}

// ================================================================================================
// Wide heads (H = 128, 192, 256): one fc1 is H*H*4 B (256 KB at H = 256), so the five of them no longer fit shared memory,
// and a warp per sample re-reading them from L2 would move ~0.8 GB per step.  A CTA of H threads instead takes a group of
// TW_G samples through the phases of tail4 together; every H x H mat-vec streams its fc1 through a double-buffered
// shared-memory k-slice (TW_KS rows) that all samples of the group consume, thread c owning output column c for every
// sample.  The per-sample vectors live in shared memory ([TW_G][H] each), the per-sample scalars are warp reductions.
// fp32 FFMA throughout, the same formulas and summation order per sample as tail4.
// ================================================================================================
// Groups of 4 samples: at B = 256 that is 64 CTAs; groups of 8 (32 CTAs, half the L2 weight traffic) measured 30 % slower.
constexpr int TW_G = 4, TW_KS = 32;
enum { V_XPI = 0, V_XVF, V_XQ1, V_XQ2, V_XT, V_XU, V_YPI, V_YVF, V_YQ1, V_YQ2, V_YT, V_YU, V_N };
// per-sample scalars, AMAX-wide blocks per action: mu (then pi), raw log_std, std, t = (u - mu) / (std + eps), the seeds of mu and
// log_std, d(-Q1(s, pi))/d pi; then one slot each
enum { SC_MU = 0, SC_LS = 8, SC_SD = 16, SC_TT = 24, SC_DMU = 32, SC_DLS = 40, SC_DPI = 48, SC_LOGP = 56, SC_ENT, SC_V, SC_VT, SC_Q1,
       SC_Q2, SC_Q1P, SC_Q2P, SC_DVF, SC_DQ1, SC_DQ2, SC_N = 72 };

template <int H>
constexpr size_t tw_smem_floats() { return 2 * (size_t)TW_KS * (H + 1) + (size_t)V_N * TW_G * H + TW_G * SC_N + 32; }

// acc[g] += sum_k x[g][k] * M[k][c] for c = threadIdx.x: M = W ([H][H] row-major fc1: forward, out[j] = sum_i a[i] W[i][j]) or,
// TR, M = W^T (backward, out[i] = sum_j dz[j] W[i][j]).  W streams through wbuf in TW_KS-deep k-slices, double-buffered
// through registers: slice s + 1 is loaded while slice s is consumed.  The caller orders x's stores before the call; the
// call ends with a barrier, so wbuf is free again and x may be overwritten afterwards.
template <int H, bool TR>
__device__ __forceinline__ void tw_matvec(const float* __restrict__ W, const float* x, float (&acc)[TW_G], float* wbuf) {
  constexpr int P = TR ? H + 1 : H;            // transposed slices: padded pitch, the scattered stores stay conflict-free
  constexpr int NS = H / TW_KS, NV = TW_KS / 4;
  const int c = threadIdx.x;
  float4 st[NV];
  auto load = [&](int s) {
    const int k0 = s * TW_KS;
#pragma unroll
    for (int m = 0; m < NV; ++m) {
      const int f = c + H * m;
      if (TR) {
        const int r = f / NV, q = f % NV;           // W[r][k0 + 4q .. + 3]
        st[m] = __ldg(reinterpret_cast<const float4*>(W + (size_t)r * H + k0 + 4 * q));
      } else {
        const int kk = f / (H / 4), c4 = f % (H / 4);
        st[m] = __ldg(reinterpret_cast<const float4*>(W + (size_t)(k0 + kk) * H + 4 * c4));
      }
    }
  };
  auto store = [&](float* buf) {
#pragma unroll
    for (int m = 0; m < NV; ++m) {
      const int f = c + H * m;
      if (TR) {
        const int r = f / NV, q = f % NV;
        buf[(4 * q) * P + r] = st[m].x; buf[(4 * q + 1) * P + r] = st[m].y;
        buf[(4 * q + 2) * P + r] = st[m].z; buf[(4 * q + 3) * P + r] = st[m].w;
      } else {
        const int kk = f / (H / 4), c4 = f % (H / 4);
        *reinterpret_cast<float4*>(buf + kk * P + 4 * c4) = st[m];
      }
    }
  };
  load(0);
  store(wbuf);
  __syncthreads();
  for (int s = 0; s < NS; ++s) {
    if (s + 1 < NS) load(s + 1);
    const float* buf = wbuf + (s & 1) * TW_KS * (H + 1);
    const int k0 = s * TW_KS;
#pragma unroll 2
    for (int kk = 0; kk < TW_KS; kk += 4) {
      float4 xv[TW_G];
#pragma unroll
      for (int g = 0; g < TW_G; ++g) xv[g] = *reinterpret_cast<const float4*>(x + g * H + k0 + kk);
      const float w0 = buf[kk * P + c], w1 = buf[(kk + 1) * P + c], w2 = buf[(kk + 2) * P + c], w3 = buf[(kk + 3) * P + c];
#pragma unroll
      for (int g = 0; g < TW_G; ++g) {
        acc[g] = fmaf(xv[g].x, w0, acc[g]); acc[g] = fmaf(xv[g].y, w1, acc[g]);
        acc[g] = fmaf(xv[g].z, w2, acc[g]); acc[g] = fmaf(xv[g].w, w3, acc[g]);
      }
    }
    if (s + 1 < NS) store(wbuf + ((s + 1) & 1) * TW_KS * (H + 1));
    __syncthreads();
  }
}

// sc[g * SC_N + slot(n)] = sum_i x(g, n)[i] * k(n)[i * kld + koff] + bias(n) for the jobs n of every sample, one warp per (g, n)
template <int H, class F>
__device__ __forceinline__ void tw_dots(int njobs, F&& job) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int p = warp; p < TW_G * njobs; p += H / 32) {
    const int g = p / njobs, n = p % njobs;
    const float* x; const float* k; int kld; float* dst; float bias;
    job(g, n, x, k, kld, dst, bias);
    float s = 0.f;
#pragma unroll
    for (int i = lane; i < H; i += 32) s = fmaf(x[i], __ldg(k + (size_t)i * kld), s);
    s = warp_sum(s);
    if (lane == 0) *dst = s + bias;
  }
}

__device__ __forceinline__ void st_planes1(uint16_t* hi, uint16_t* lo, size_t o, float v) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[o] = __bfloat16_as_ushort(h);
  lo[o] = __bfloat16_as_ushort(__float2bfloat16_rn(v - __bfloat162float(h)));
}

template <int H>
__global__ void __launch_bounds__(H) tailw_kernel(TailArgs t) {
  extern __shared__ __align__(16) float smem[];
  float* wbuf = smem;
  float* V = wbuf + 2 * TW_KS * (H + 1);
  float* sc = V + V_N * TW_G * H;
  float* red = sc + TW_G * SC_N;                  // [MET_COUNT + 1] loss / metric sums of the group
  auto vec = [&](int v, int g) { return V + (v * TW_G + g) * H; };
  const int c = threadIdx.x, A = t.A, b_base = blockIdx.x * TW_G;
  pdl_trigger();
  pdl_wait();
  if (c <= MET_COUNT) red[c] = 0.f;
  const float invB = 1.0f / (float)t.grad_scale_B;
  const float log_alpha = t.log_alpha[0];
  const float alpha = expf(log_alpha);
  const float* K1[S_NW] = {t.pi.k1, t.vf.k1, t.q1.k1, t.q2.k1, t.vt.k1};
  float acc[TW_G];

  // ---- fc0 activations at the replay action (rows past the batch are zeros and contribute nothing)
  {
    const float b0p = t.pi.b0[c], b0v = t.vf.b0[c], b0q1 = t.q1.b0[c], b0q2 = t.q2.b0[c], b0t = t.vt.b0[c];
    for (int g = 0; g < TW_G; ++g) {
      const int b = b_base + g;
      const bool ok = b < t.B;
      const size_t ov = (size_t)b * t.z0v_ld + c;
      const float a0p = ok ? fmaxf(t.z0_pi[(size_t)b * H + c] + b0p, 0.f) : 0.f;
      const float a0v = ok ? fmaxf(t.z0_vf[ov] + b0v, 0.f) : 0.f;
      const float a0q1 = ok ? fmaxf(t.z0_q1[ov] + b0q1, 0.f) : 0.f;
      const float a0q2 = ok ? fmaxf(t.z0_q2[ov] + b0q2, 0.f) : 0.f;
      vec(V_XPI, g)[c] = a0p; vec(V_XVF, g)[c] = a0v; vec(V_XQ1, g)[c] = a0q1; vec(V_XQ2, g)[c] = a0q2;
      vec(V_XT, g)[c] = ok ? fmaxf(t.z0_vt[(size_t)b * H + c] + b0t, 0.f) : 0.f;
      if (ok) {
        const size_t o = (size_t)b * H + c;
        t.a0_pi[o] = a0p; t.a0_vf[o] = a0v; t.a0_q1[o] = a0q1; t.a0_q2[o] = a0q2;
      }
    }
  }
  __syncthreads();
  // ---- fc1 forward of the five heads
  {
    const int xin[S_NW] = {V_XPI, V_XVF, V_XQ1, V_XQ2, V_XT}, yout[S_NW] = {V_YPI, V_YVF, V_YQ1, V_YQ2, V_YT};
    const float* b1s[S_NW] = {t.pi.b1, t.vf.b1, t.q1.b1, t.q2.b1, t.vt.b1};
    for (int w = 0; w < S_NW; ++w) {
      const float bias = b1s[w][c];
#pragma unroll
      for (int g = 0; g < TW_G; ++g) acc[g] = bias;
      tw_matvec<H, false>(K1[w], vec(xin[w], 0), acc, wbuf);
#pragma unroll
      for (int g = 0; g < TW_G; ++g) vec(yout[w], g)[c] = fmaxf(acc[g], 0.f);
    }
  }
  __syncthreads();
  // ---- output layers: mu, log_std (raw), v, v_targ, q1, q2
  tw_dots<H>(2 * A + 4, [&](int g, int n, const float*& x, const float*& k, int& kld, float*& dst, float& bias) {
    if (n < 2 * A) {
      const int a = n % A;
      const bool mu = n < A;
      x = vec(V_YPI, g); k = (mu ? t.pi.ko : t.ksig) + a; kld = A;
      dst = sc + g * SC_N + (mu ? SC_MU : SC_LS) + a; bias = (mu ? t.pi.bo : t.bsig)[a];
      return;
    }
    const int m = n - 2 * A;                   // 0 vf, 1 target vf, 2 qf1, 3 qf2
    const HeadW* hw = m == 0 ? &t.vf : m == 1 ? &t.vt : m == 2 ? &t.q1 : &t.q2;
    x = vec(m == 0 ? V_YVF : m == 1 ? V_YT : m == 2 ? V_YQ1 : V_YQ2, g); k = hw->ko; kld = 1;
    dst = sc + g * SC_N + SC_V + m; bias = hw->bo[0];
  });
  __syncthreads();
  // ---- actor outputs (one thread per sample)
  if (c < TW_G) {
    const int b = b_base + c;
    float* s = sc + c * SC_N;
    float logp = 0.f, ent = 0.f;
    for (int a = 0; a < A; ++a) {
      const float e = b < t.B ? t.eps[b * A + a] : 0.f;
      const float mu = s[SC_MU + a];
      const float ls = fminf(fmaxf(s[SC_LS + a], LS_MIN), LS_MAX);
      const float sd = expf(ls);
      const float u = mu + e * sd;
      const float tt = (u - mu) / (sd + EPSF);
      const float pi = tanhf(u);
      logp += -0.5f * (tt * tt + 2.f * ls + 1.8378770664093453f) - logf(1.f - pi * pi + EPSF);
      ent += ls + 1.4189385332046727f;
      s[SC_SD + a] = sd; s[SC_TT + a] = tt; s[SC_MU + a] = pi;      // mu is not needed past here: its slot holds pi
      if (t.pi_out && b < t.B) t.pi_out[b * A + a] = pi;
    }
    s[SC_LOGP] = logp; s[SC_ENT] = ent;
  }
  __syncthreads();
  // ---- qf1, qf2 at pi: z0(pi) = z0(a) + (pi - a) K0[action rows]
  {
    const float b0q1 = t.q1.b0[c], b0q2 = t.q2.b0[c];
    for (int g = 0; g < TW_G; ++g) {
      const int b = b_base + g;
      float x1 = 0.f, x2 = 0.f;
      if (b < t.B) {
        const size_t ov = (size_t)b * t.z0v_ld + c;
        float z1 = t.z0_q1[ov], z2 = t.z0_q2[ov];
        for (int a = 0; a < A; ++a) {
          const float dlt = sc[g * SC_N + SC_MU + a] - t.act[(size_t)b * t.act_stride + a];
          const size_t ro = (size_t)(t.feat_dim + a) * H + c;
          z1 = fmaf(dlt, t.q1.k0[ro], z1); z2 = fmaf(dlt, t.q2.k0[ro], z2);
        }
        x1 = fmaxf(z1 + b0q1, 0.f); x2 = fmaxf(z2 + b0q2, 0.f);
      }
      vec(V_XT, g)[c] = x1; vec(V_XU, g)[c] = x2;
    }
  }
  __syncthreads();
  {
    const float bq1 = t.q1.b1[c], bq2 = t.q2.b1[c];
#pragma unroll
    for (int g = 0; g < TW_G; ++g) acc[g] = bq1;
    tw_matvec<H, false>(t.q1.k1, vec(V_XT, 0), acc, wbuf);
#pragma unroll
    for (int g = 0; g < TW_G; ++g) vec(V_YT, g)[c] = fmaxf(acc[g], 0.f);      // (target vf activations are dead)
#pragma unroll
    for (int g = 0; g < TW_G; ++g) acc[g] = bq2;
    tw_matvec<H, false>(t.q2.k1, vec(V_XU, 0), acc, wbuf);
#pragma unroll
    for (int g = 0; g < TW_G; ++g) vec(V_YU, g)[c] = fmaxf(acc[g], 0.f);
  }
  __syncthreads();
  tw_dots<H>(2, [&](int g, int n, const float*& x, const float*& k, int& kld, float*& dst, float& bias) {
    const HeadW* hw = n == 0 ? &t.q1 : &t.q2;
    x = vec(n == 0 ? V_YT : V_YU, g); k = hw->ko; kld = 1; dst = sc + g * SC_N + SC_Q1P + n; bias = hw->bo[0];
  });
  __syncthreads();
  // ---- losses, metrics and the value / Q backward seeds (one thread per sample)
  if (c < TW_G) {
    const int b = b_base + c;
    float* s = sc + c * SC_N;
    float dvf = 0.f, dq1 = 0.f, dq2 = 0.f;
    if (b < t.B) {
      const float logp = s[SC_LOGP], q1p = s[SC_Q1P], q2p = s[SC_Q2P], v = s[SC_V], v_targ = s[SC_VT];
      atomicAdd(&red[MET_POLICY_LOSS], (alpha * logp - q1p) * invB);
      atomicAdd(&red[MET_ENT_COEF_LOSS], -log_alpha * (logp + t.target_entropy) * invB);
      atomicAdd(&red[MET_ENTROPY], s[SC_ENT] * invB);
      atomicAdd(&red[MET_MEAN_LOGP], logp * invB);
      atomicAdd(&red[MET_COUNT], -(logp + t.target_entropy) * invB);
      const float v_backup = fminf(q1p, q2p) - alpha * logp;
      const float ev = v - v_backup;
      atomicAdd(&red[MET_VALUE_LOSS], 0.5f * ev * ev * invB);
      atomicAdd(&red[MET_MEAN_V], v * invB);
      dvf = ev * invB;
      const float q_backup = t.rew[b] + (1.f - t.done[b]) * t.gamma * v_targ;
      const float e1 = s[SC_Q1] - q_backup, e2 = s[SC_Q2] - q_backup;
      atomicAdd(&red[MET_QF1_LOSS], 0.5f * e1 * e1 * invB);
      atomicAdd(&red[MET_QF2_LOSS], 0.5f * e2 * e2 * invB);
      atomicAdd(&red[MET_MEAN_Q1], s[SC_Q1] * invB);
      atomicAdd(&red[MET_MEAN_Q2], s[SC_Q2] * invB);
      dq1 = e1 * invB; dq2 = e2 * invB;
      if (t.per_sample) {
        const int B = t.B;
        t.per_sample[b] = s[SC_Q1]; t.per_sample[B + b] = s[SC_Q2]; t.per_sample[2 * B + b] = v; t.per_sample[3 * B + b] = logp;
        t.per_sample[4 * B + b] = v_targ; t.per_sample[5 * B + b] = q1p; t.per_sample[6 * B + b] = q2p;
      }
    }
    s[SC_DVF] = dvf; s[SC_DQ1] = dq1; s[SC_DQ2] = dq2;
  }
  // d(-Q1(s, pi))/d a1 at pi -> V_YU (the qf2-at-pi activations are dead)
  {
    const float k = t.q1.ko[c];
    for (int g = 0; g < TW_G; ++g)
      vec(V_YU, g)[c] = (b_base + g < t.B && vec(V_YT, g)[c] > 0.f) ? -invB * k : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int g = 0; g < TW_G; ++g) acc[g] = 0.f;
  tw_matvec<H, true>(t.q1.k1, vec(V_YU, 0), acc, wbuf);
#pragma unroll
  for (int g = 0; g < TW_G; ++g) vec(V_XU, g)[c] = vec(V_XT, g)[c] > 0.f ? acc[g] : 0.f;      // dz0 of qf1 at pi
  __syncthreads();
  // dpi = dz0(pi) . K0[action rows]^T
  tw_dots<H>(A, [&](int g, int n, const float*& x, const float*& k, int& kld, float*& dst, float& bias) {
    x = vec(V_XU, g); k = t.q1.k0 + (size_t)(t.feat_dim + n) * H; kld = 1; dst = sc + g * SC_N + SC_DPI + n; bias = 0.f;
  });
  __syncthreads();
  // ---- actor backward seeds (one thread per sample)
  if (c < TW_G) {
    const int b = b_base + c;
    float* s = sc + c * SC_N;
    for (int a = 0; a < A; ++a) {
      float dmu = 0.f, dls = 0.f;
      if (b < t.B) {
        const float e = t.eps[b * A + a], pi = s[SC_MU + a], sd = s[SC_SD + a], tt = s[SC_TT + a], ls_raw = s[SC_LS + a];
        const float one_m = 1.f - pi * pi;
        const float du = (alpha * invB) * 2.f * pi * one_m / (one_m + EPSF) + s[SC_DPI + a] * one_m;
        dmu = du;
        const float spe = sd + EPSF;
        const float d = du * e * sd + (alpha * invB) * (-tt * e * sd * EPSF / (spe * spe) - 1.f);
        dls = (ls_raw >= LS_MIN && ls_raw <= LS_MAX) ? d : 0.f;
      }
      s[SC_DMU + a] = dmu; s[SC_DLS + a] = dls;
    }
  }
  __syncthreads();
  // ---- fc1 pre-activation gradients (column c of every sample) and the output-layer gradients of the group
  float gk_mu[AMAX], gk_sig[AMAX];
  float gko_vf = 0.f, gko_q1 = 0.f, gko_q2 = 0.f;
  {
    float kmu[AMAX], ksg[AMAX];
#pragma unroll
    for (int a = 0; a < AMAX; ++a) {
      kmu[a] = a < A ? t.pi.ko[c * A + a] : 0.f; ksg[a] = a < A ? t.ksig[c * A + a] : 0.f;
      gk_mu[a] = 0.f; gk_sig[a] = 0.f;
    }
    const float kvf = t.vf.ko[c], kq1 = t.q1.ko[c], kq2 = t.q2.ko[c];
    for (int g = 0; g < TW_G; ++g) {
      const int b = b_base + g;
      const float* s = sc + g * SC_N;
      const float gv = vec(V_YPI, g)[c];
      float dg = 0.f;
#pragma unroll
      for (int a = 0; a < AMAX; ++a) {
        if (a < A) {
          const float dmu = s[SC_DMU + a], dls = s[SC_DLS + a];
          gk_mu[a] = fmaf(gv, dmu, gk_mu[a]); gk_sig[a] = fmaf(gv, dls, gk_sig[a]);
          dg += dmu * kmu[a] + dls * ksg[a];
        }
      }
      const float dz_pi = gv > 0.f ? dg : 0.f;
      float* yvf = vec(V_YVF, g); float* yq1 = vec(V_YQ1, g); float* yq2 = vec(V_YQ2, g);
      const float a1v = yvf[c], a1q1 = yq1[c], a1q2 = yq2[c];
      const float dvf = s[SC_DVF], dq1 = s[SC_DQ1], dq2 = s[SC_DQ2];
      gko_vf = fmaf(a1v, dvf, gko_vf); gko_q1 = fmaf(a1q1, dq1, gko_q1); gko_q2 = fmaf(a1q2, dq2, gko_q2);
      const float dz_vf = a1v > 0.f ? dvf * kvf : 0.f, dz_q1 = a1q1 > 0.f ? dq1 * kq1 : 0.f, dz_q2 = a1q2 > 0.f ? dq2 * kq2 : 0.f;
      vec(V_YT, g)[c] = dz_pi; yvf[c] = dz_vf; yq1[c] = dz_q1; yq2[c] = dz_q2;      // in place: column c is this thread's own
      if (b < t.B) {
        const size_t o = (size_t)b * H + c;
        t.dz1_pi[o] = dz_pi; t.dz1_vf[o] = dz_vf; t.dz1_q1[o] = dz_q1; t.dz1_q2[o] = dz_q2;
      }
    }
  }
  __syncthreads();
  // ---- fc1^T backward of pi, vf, qf1, qf2 -> dz0 (fp32 and, for engine v2, BF16 hi / lo planes)
  {
    const int yin[4] = {V_YT, V_YVF, V_YQ1, V_YQ2}, xin[4] = {V_XPI, V_XVF, V_XQ1, V_XQ2};
    const float* W[4] = {t.pi.k1, t.vf.k1, t.q1.k1, t.q2.k1};
    for (int w = 0; w < 4; ++w) {
#pragma unroll
      for (int g = 0; g < TW_G; ++g) acc[g] = 0.f;
      tw_matvec<H, true>(W[w], vec(yin[w], 0), acc, wbuf);
      for (int g = 0; g < TW_G; ++g) {
        const int b = b_base + g;
        if (b >= t.B) break;
        const float dz0 = vec(xin[w], g)[c] > 0.f ? acc[g] : 0.f;
        if (w == 0) {
          const size_t o = (size_t)b * H + c;
          t.dz0_pi[o] = dz0;
          if (t.dz0_pi_p[0]) st_planes1(t.dz0_pi_p[0], t.dz0_pi_p[1], o, dz0);
        } else {
          const size_t o = (size_t)b * 3 * H + (w - 1) * H + c;
          t.dz0_v3[o] = dz0;
          if (t.dz0_v3_p[0]) st_planes1(t.dz0_v3_p[0], t.dz0_v3_p[1], o, dz0);
        }
      }
    }
  }
  // ---- the group's gradient contributions (tw_matvec ended with a barrier: red is complete)
#pragma unroll
  for (int a = 0; a < AMAX; ++a)
    if (a < A) { atomicAdd(t.g_pi.ko + c * A + a, gk_mu[a]); atomicAdd(t.g_ksig + c * A + a, gk_sig[a]); }
  atomicAdd(t.g_vf.ko + c, gko_vf); atomicAdd(t.g_q1.ko + c, gko_q1); atomicAdd(t.g_q2.ko + c, gko_q2);
  if (c < A) {
    float sm = 0.f, ss = 0.f;
    for (int g = 0; g < TW_G; ++g) { sm += sc[g * SC_N + SC_DMU + c]; ss += sc[g * SC_N + SC_DLS + c]; }
    atomicAdd(t.g_pi.bo + c, sm); atomicAdd(t.g_bsig + c, ss);
  }
  if (c == 0) {
    float sv = 0.f, s1 = 0.f, s2 = 0.f;
    for (int g = 0; g < TW_G; ++g) { sv += sc[g * SC_N + SC_DVF]; s1 += sc[g * SC_N + SC_DQ1]; s2 += sc[g * SC_N + SC_DQ2]; }
    atomicAdd(t.g_vf.bo, sv); atomicAdd(t.g_q1.bo, s1); atomicAdd(t.g_q2.bo, s2);
    atomicAdd(t.g_log_alpha, red[MET_COUNT]);
  }
  if (c < MET_GN_PI) atomicAdd(t.metrics + c, red[c]);
}

// policy inference at H >= 128: tanh(mu) or tanh(mu + eps * std) for TW_G rows per CTA, fc1 streamed as in tailw_kernel
template <int H>
__global__ void __launch_bounds__(H) actw_kernel(TailArgs t, int n, int deterministic, float* act_out) {
  extern __shared__ __align__(16) float smem[];
  float* wbuf = smem;
  float* X = wbuf + 2 * TW_KS * (H + 1);
  float* Y = X + TW_G * H;
  float* sc = Y + TW_G * H;                       // [TW_G][2 * AMAX]: mu, log_std
  const int c = threadIdx.x, A = t.A, b_base = blockIdx.x * TW_G;
  const float b0 = t.pi.b0[c];
  for (int g = 0; g < TW_G; ++g) {
    const int b = b_base + g;
    X[g * H + c] = b < n ? fmaxf(t.z0_pi[(size_t)b * H + c] + b0, 0.f) : 0.f;
  }
  __syncthreads();
  float acc[TW_G];
  const float b1 = t.pi.b1[c];
#pragma unroll
  for (int g = 0; g < TW_G; ++g) acc[g] = b1;
  tw_matvec<H, false>(t.pi.k1, X, acc, wbuf);
#pragma unroll
  for (int g = 0; g < TW_G; ++g) Y[g * H + c] = fmaxf(acc[g], 0.f);
  __syncthreads();
  tw_dots<H>(2 * A, [&](int g, int m, const float*& x, const float*& k, int& kld, float*& dst, float& bias) {
    const int a = m % A;
    const bool mu = m < A;
    x = Y + g * H; k = (mu ? t.pi.ko : t.ksig) + a; kld = A; dst = sc + g * 2 * AMAX + (mu ? 0 : AMAX) + a; bias = (mu ? t.pi.bo : t.bsig)[a];
  });
  __syncthreads();
  if (c < TW_G * A) {
    const int g = c / A, a = c % A, b = b_base + g;
    if (b < n) {
      float u = sc[g * 2 * AMAX + a];
      if (!deterministic) u += t.eps[b * A + a] * expf(fminf(fmaxf(sc[g * 2 * AMAX + AMAX + a], LS_MIN), LS_MAX));
      act_out[b * A + a] = tanhf(u);
    }
  }
}

template <int H>
size_t tailw_smem() { return sizeof(float) * tw_smem_floats<H>(); }
template <int H>
size_t actw_smem() { return sizeof(float) * (2 * (size_t)TW_KS * (H + 1) + 2 * TW_G * H + TW_G * 2 * AMAX); }

// The opt-in to more than 48 KB of dynamic shared memory is a property of the kernel on ONE device: it is set the first time a
// kernel is launched on each device (done: one bit per device ordinal) and its failure is returned.
template <class K>
cudaError_t smem_optin(K* fn, size_t bytes, unsigned long long& done) {
  int dev = 0;
  if (cudaError_t e = cudaGetDevice(&dev)) return e;
  const unsigned long long bit = dev < 64 ? 1ull << dev : 0ull;
  if (done & bit) return cudaSuccess;
  if (cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes)) return e;
  done |= bit;
  return cudaSuccess;
}

template <int H>
cudaError_t tailw_launch(const TailArgs& a, cudaStream_t s, bool pdl) {
  static unsigned long long done = 0;
  if (cudaError_t e = smem_optin(tailw_kernel<H>, tailw_smem<H>(), done)) return e;
  return launch_pdl(tailw_kernel<H>, dim3((a.B + TW_G - 1) / TW_G), dim3(H), tailw_smem<H>(), s, pdl, a);
}
template <int H>
cudaError_t actw_launch(const TailArgs& t, int n, int deterministic, float* act_out, cudaStream_t s) {
  static unsigned long long done = 0;
  if (cudaError_t e = smem_optin(actw_kernel<H>, actw_smem<H>(), done)) return e;
  actw_kernel<H><<<(n + TW_G - 1) / TW_G, H, actw_smem<H>(), s>>>(t, n, deterministic, act_out);
  return cudaPeekAtLastError();
}

}  // namespace

cudaError_t act_launch(const TailArgs& t, int n, int deterministic, float* act_out, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  switch (t.H) {
    case 128: return actw_launch<128>(t, n, deterministic, act_out, s);
    case 192: return actw_launch<192>(t, n, deterministic, act_out, s);
    case 256: return actw_launch<256>(t, n, deterministic, act_out, s);
  }
  act_kernel<<<(n + WARPS - 1) / WARPS, WARPS * 32, 0, s>>>(t, n, deterministic, act_out);
  return cudaPeekAtLastError();
}

namespace {
// grid (9 + H/64, 4 heads, HW_KSPLIT batch slices x H/64 column blocks), 256 threads: x = 0..8 -> rows [64x, 64x + 64) of the
// fc0 kernel gradient X0^T . dz0 (x = 0 also the fc0 bias gradient: column sums of dz0), x = 9.. -> row block x - 9 of the fc1
// kernel gradient a0^T . dz1 (x = 9 also the fc1 bias); every CTA covers 64 output columns.  Every CTA
// reduces its batch slice in chunks of 32 samples through shared memory (4 x 4 outputs per thread) and accumulates into the
// zeroed gradient arena with red.add.
constexpr int HW_KSPLIT = 4;
__global__ void __launch_bounds__(256) heads_wgrad_kernel(const HeadsWgradArgs a) {
  __shared__ __align__(16) float As[32][64], Bs[32][64];
  const int q = blockIdx.y, rb = blockIdx.x, tid = threadIdx.x, tx = tid & 15, ty = tid >> 4, H = a.H;
  const bool fc1 = rb >= 9, sums = rb == 0 || rb == 9;
  const int M = fc1 ? H : a.M0[q], row0 = (fc1 ? rb - 9 : rb) * 64, n0 = (blockIdx.z / HW_KSPLIT) * 64;
  if (row0 >= M) return;
  const float* __restrict__ X = fc1 ? a.a0[q] : a.X0[q];
  const float* __restrict__ D = (fc1 ? a.dz1[q] : a.dz0[q]) + n0;
  const int xld = fc1 ? H : a.x0_ld, dld = fc1 ? H : a.dz0_ld[q];
  const int per = (a.B + HW_KSPLIT - 1) / HW_KSPLIT, b0 = (blockIdx.z % HW_KSPLIT) * per, b1 = min(a.B, b0 + per);
  float acc[4][4] = {};
  float cs = 0.f;                         // bias sum: column n0 + tid (x == 0: fc0 bias from dz0, x == 9: fc1 bias from dz1)
  for (int bb = b0; bb < b1; bb += 32) {
    for (int i = tid; i < 32 * 64; i += 256) {
      const int k = i >> 6, c = i & 63, b = bb + k;
      const bool ok = b < b1;
      As[k][c] = (ok && row0 + c < M) ? X[(size_t)b * xld + row0 + c] : 0.f;
      Bs[k][c] = ok ? D[(size_t)b * dld + c] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < 32; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&As[k][4 * ty]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][4 * tx]);
      const float ar[4] = {av.x, av.y, av.z, av.w}, br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
    }
    if (sums && tid < 64) {
#pragma unroll 8
      for (int k = 0; k < 32; ++k) cs += Bs[k][tid];
    }
    __syncthreads();
  }
  float* __restrict__ G = (fc1 ? a.g_k1[q] : a.g_k0[q]) + n0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = row0 + 4 * ty + i;
    if (r < M)
      asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(G + (size_t)r * H + 4 * tx), "f"(acc[i][0]), "f"(acc[i][1]), "f"(acc[i][2]),
                   "f"(acc[i][3])
                   : "memory");
  }
  if (sums && tid < 64) atomicAdd((fc1 ? a.g_b1[q] : a.g_b0[q]) + n0 + tid, cs);
}
}  // namespace

void heads_wgrad_launch(const HeadsWgradArgs& a, cudaStream_t s) {
  heads_wgrad_kernel<<<dim3(9 + a.H / 64, 4, HW_KSPLIT * (a.H / 64)), 256, 0, s>>>(a);
}

static size_t tail_smem(int A) {
  return sizeof(float) * (S_NW * H * LD + 2 * H * A + 2 * A + 3 * (H + 1) + MET_COUNT + 1 + 8 +
                          /* staged small parameters */ (S_NW * 2 * H + 2 * H * A + 2 * A + 4 * (H + 1) + 2 * A * H + 8) +
                          /* tail4 scratch */ 64);
}

cudaError_t tail_launch(const TailArgs& a, cudaStream_t s, bool pdl) {
  switch (a.H) {
    case 128: return tailw_launch<128>(a, s, pdl);
    case 192: return tailw_launch<192>(a, s, pdl);
    case 256: return tailw_launch<256>(a, s, pdl);
  }
  static unsigned long long done = 0;
  if (cudaError_t e = smem_optin(tail4_kernel, tail_smem(AMAX), done)) return e;
  const int grid = (a.B + 1) / 2;             // four warps per sample, two samples per CTA
  return launch_pdl(tail4_kernel, dim3(grid), dim3(WARPS * 32), tail_smem(a.A), s, pdl, a);
}

}  // namespace b2g
