// Engine v2: the CNN / head contractions of the SAC step on the TMA-fed wgmma engine (cg.cu).
//
// This file owns (i) the BF16 plane tensors the engine reads and writes, (ii) the tensor-map VIEWS that turn NHWC
// activation planes into implicit-im2col / shifted-window / zero-bordered operand tiles (one map per tensor: plane = outermost
// dimension), (iii) the problem lists of every layer group and the two FUSED launches built from them (forward chain, backward
// chain: fuse_groups wires each consumer problem to the producer tiles it reads) and (iv) the HBM-bound helper kernels around them:
//   gather2_kernel : replay slot draw + gather of replay frames (compact rows, replay.cu) + float64 VecNormalize +
//                    clip + /255 (replay.cu semantics, [SB2] ReplayBuffer.sample(env=VecNormalize), observation_input(scale=True)),
//                    the 3-plane BF16 split, stored space-to-depth (S, below) so that conv1's 8x8 stride-4 patches become a
//                    2x2 stride-1 window over S: four shifted boxes of a monotonic tensor-map view;
//   planes2_kernel : weights -> BF16 planes in the layouts the tensor maps expect (transposed / packed per consumer).
// The bias gradients of the conv and cnn_fc1 layers come from the DGRAD epilogues of cg.cu (column sums of the gradient maps).
// Reference shapes: custom_obs_policy.py:34-40 (conv 8x8/4 -> 4x4/2 -> 3x3/1, fc 1024->512), SURVEY.md Appendix A.
#include <cuda_bf16.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "sac_internal.cuh"

namespace b2g {
namespace {

// ------------------------------------------------------------------------------------------------ gather2
struct Gather2Args {
  GatherArgs g;                 // sources, statistics, F rows (fp32), reward / done outputs, slot draw
  uint16_t* s1[2][3];           // space-to-depth images [B][16][16][4][4][Cp] (obs, next_obs) x 3 planes
  uint16_t* fp[3][3];           // feature-row planes [net][plane] [B][KF]
  int KF;
};

__device__ __forceinline__ void split3(float y, uint16_t& p0, uint16_t& p1, uint16_t& p2) {
  const __nv_bfloat16 h0 = __float2bfloat16_rn(y);
  const float r1 = y - __bfloat162float(h0);
  const __nv_bfloat16 h1 = __float2bfloat16_rn(r1);
  const float r2 = r1 - __bfloat162float(h1);
  p0 = __bfloat16_as_ushort(h0); p1 = __bfloat16_as_ushort(h1); p2 = __bfloat16_as_ushort(__float2bfloat16_rn(r2));
}

// Half a 4x4 block of the space-to-depth image S[Y][X][b][c][ci] (pixel (4Y + b, 4X + c), channel ci < CP; ci >= Ci is a zero
// pad): image rows b = 2h, 2h + 1 of the block, 4 pixels each.  The 4 CP values of a row are contiguous in S (8 CP bytes) and the
// threads of a warp cover consecutive half blocks, so its stores fill whole sectors.  Normalise / clip / scale / split as the
// round-1 gather does, element by element.
template <int Ci>
__device__ __forceinline__ void s2d_half_block(const Gather2Args& a, const unsigned char* __restrict__ src, int it, int which, size_t b) {
  constexpr int CP = s2d_channels(Ci);
  const GatherArgs& g = a.g;
  const int npx = g.H * g.W * Ci;
  const int h = it & 1, X = (it >> 1) & 15, Y = it >> 5;
  const double clip_obs = g.normc[1];
  const bool norm_obs = g.normc[3] != 0.0;
  const float scale = g.scale;
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int e0 = ((4 * Y + 2 * h + rr) * g.W + 4 * X) * Ci;      // 4 pixels x Ci channels, a multiple of 4 elements
    float y[4 * Ci];
#pragma unroll
    for (int q = 0; q < Ci; ++q) {
      const int e = e0 + 4 * q;
      const float4 v = frame_load4(src, g.fmt, npx, Ci, e);
      float t[4] = {v.x, v.y, v.z, v.w};
      if (norm_obs) {
        const double2 m0 = *reinterpret_cast<const double2*>(g.mean + e), m1 = *reinterpret_cast<const double2*>(g.mean + e + 2);
        const double2 i0 = *reinterpret_cast<const double2*>(g.var + e), i1 = *reinterpret_cast<const double2*>(g.var + e + 2);
        t[0] = (float)fmin(fmax(((double)t[0] - m0.x) * i0.x, -clip_obs), clip_obs);
        t[1] = (float)fmin(fmax(((double)t[1] - m0.y) * i0.y, -clip_obs), clip_obs);
        t[2] = (float)fmin(fmax(((double)t[2] - m1.x) * i1.x, -clip_obs), clip_obs);
        t[3] = (float)fmin(fmax(((double)t[3] - m1.y) * i1.y, -clip_obs), clip_obs);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) y[4 * q + j] = t[j];
    }
    uint32_t p[3][2 * CP];                                   // the row's 4 CP values per plane, packed in pairs
#pragma unroll
    for (int k = 0; k < 4 * CP; k += 2) {
      uint16_t q[3][2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int c = (k + u) / CP, ci = (k + u) % CP;
        if (ci < Ci) split3(y[c * Ci + ci] / scale, q[0][u], q[1][u], q[2][u]);
        else q[0][u] = q[1][u] = q[2][u] = 0;
      }
#pragma unroll
      for (int pl = 0; pl < 3; ++pl) p[pl][k / 2] = (uint32_t)q[pl][0] | ((uint32_t)q[pl][1] << 16);
    }
    const size_t o = b * 4096 * CP + (size_t)((Y * 16 + X) * 16 + 4 * (2 * h + rr)) * CP;
#pragma unroll
    for (int pl = 0; pl < 3; ++pl) {
      if constexpr (CP == 1) {
        *reinterpret_cast<uint2*>(a.s1[which][pl] + o) = make_uint2(p[pl][0], p[pl][1]);
      } else {
        uint4* d = reinterpret_cast<uint4*>(a.s1[which][pl] + o);
        d[0] = make_uint4(p[pl][0], p[pl][1], p[pl][2], p[pl][3]);
        d[1] = make_uint4(p[pl][4], p[pl][5], p[pl][6], p[pl][7]);
      }
    }
  }
}

// one CTA per (sample, obs | next_obs), one thread per half 4x4 block of the 64 x 64 image (Ci image channels)
template <int Ci>
__global__ void __launch_bounds__(512) gather2_kernel(Gather2Args a) {
  const GatherArgs& g = a.g;
  const int b = blockIdx.x, which = blockIdx.y, tid = threadIdx.x;
  const int HW = g.H * g.W, npx = HW * Ci;
  const int Ec = npx + 4;                                  // compact replay row: image planes | actuator value | 3 pad floats
  long long slot = b;
  if (g.indices) slot = g.indices[b];
  else if (g.rng_counters) {
    slot = philox_slot(g.seed, (unsigned long long)g.rng_counters[4], b, (unsigned long long)g.rng_counters[5]);
    if (g.ring_cap > 0) slot = ring_slot(g.rng_counters[6], (int)slot, g.ring_cap);
    if (g.indices_out && which == 0 && tid == 0) g.indices_out[b] = (int)slot;
  }
  const unsigned char* __restrict__ src =
      g.obs_frame ? g.frames + (size_t)(which ? g.next_frame : g.obs_frame)[slot] * g.frame_bytes
                  : reinterpret_cast<const unsigned char*>((which ? g.next_obs : g.obs) + (size_t)slot * Ec);
  const double clip_obs = g.normc[1];
  const bool norm_obs = g.normc[3] != 0.0;
  const float scale = g.scale;
  for (int it = tid; it < 512; it += blockDim.x) s2d_half_block<Ci>(a, src, it, which, b);
  if (tid == 0 && g.feat_col >= 0) {                         // direct feature -> column 512 of the feature rows
    float yy = frame_elem(src, g.fmt, npx, Ci, npx);
    if (norm_obs) yy = (float)fmin(fmax(((double)yy - g.mean[npx]) * g.var[npx], -clip_obs), clip_obs);
    yy = yy / scale;
    uint16_t p0, p1, p2;
    split3(yy, p0, p1, p2);
    const size_t fo = (size_t)b * g.FS + g.feat_col, po = (size_t)b * a.KF + g.feat_col;
    if (which) { g.F_t[fo] = yy; a.fp[2][0][po] = p0; a.fp[2][1][po] = p1; a.fp[2][2][po] = p2; }
    else {
      g.F_pi[fo] = yy; g.F_v[fo] = yy;
      a.fp[0][0][po] = p0; a.fp[0][1][po] = p1; a.fp[0][2][po] = p2;
      a.fp[1][0][po] = p0; a.fp[1][1][po] = p1; a.fp[1][2][po] = p2;
    }
  }
  if (which == 0 && g.act) {
    const int feat_dim = g.act_col;
    if (tid < g.n_act) {
      const float av = g.act[slot * g.n_act + tid];
      g.F_v[(size_t)b * g.FS + feat_dim + tid] = av;
      uint16_t p0, p1, p2;
      split3(av, p0, p1, p2);
      const size_t po = (size_t)b * a.KF + feat_dim + tid;
      a.fp[1][0][po] = p0; a.fp[1][1][po] = p1; a.fp[1][2][po] = p2;
    }
    if (tid == 32) {
      float r = g.rew[slot];
      if (g.normc[4] != 0.0) r = (float)fmin(fmax((double)r * g.normc[0], -g.normc[2]), g.normc[2]);
      g.rew_out[b] = r;
      g.done_out[b] = g.done[slot];
    }
  }
}

// ------------------------------------------------------------------------------------------------ planes2
struct Plane2Job {
  const float* src;          // [R][N] row-major fp32
  uint16_t* dst[3];          // plane bases (np of them)
  int R, N, np;
  int transpose;             // 1: dst[(n + off0) * ld + r]   0: dst[r * ld + n + off0]
  int ld, off0;
  int k1_ci;                 // > 0 (transposed conv1 weights of k1_ci channels): row r goes to K row conv1_krow(r, k1_ci)
  int tile_start;
};

// 64 (r) x 32 P2_SUB (n) source strip per CTA, as P2_SUB sub-tiles of 64 x 32 whose loads are all in flight before the first
// is used: about 30 MB move per step, and 64 x 32 tiles (2 float4 loads per thread) left it latency-bound at under 1 TB/s.
// Loads are float4 along n; the transposed copy is written as 16-byte runs of 8 consecutive r values per plane (the 2-byte
// scattered stores of the first version made this the longest leaf kernel).  CTA cta0 + blockIdx.x of the job table.  Jobs
// narrower than the strip (conv1: N = 32; fc0 at H = 64; conv2 / conv3: N = 64) leave sub-tiles idle: bounds-checked, no loads.
constexpr int P2_SUB = 4;
__global__ void __launch_bounds__(256) planes2_kernel(const Plane2Job* __restrict__ jobs, const int* __restrict__ cta_job, int cta0) {
  __shared__ float tile[P2_SUB][64][33];
  // (the job of a CTA comes from a table: walking the job list cost up to 30 DEPENDENT global loads before the first useful one)
  const int cta = cta0 + blockIdx.x;
  const Plane2Job job = jobs[cta_job[cta]];
  const int t = cta - job.tile_start;
  const int strips_n = (job.N + 32 * P2_SUB - 1) / (32 * P2_SUB);
  const int r0 = (t / strips_n) * 64, nb = (t % strips_n) * 32 * P2_SUB;
  const int tid = threadIdx.x;
  // ---- load P2_SUB x (64 x 32): 8 float4 per row of a sub-tile, 2 passes of 32 rows
  const bool vec_ok = (job.N & 3) == 0;
  float4 v[P2_SUB][2];
#pragma unroll
  for (int q = 0; q < P2_SUB; ++q)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int i = tid + 256 * j, r = r0 + (i >> 3), n = nb + 32 * q + 4 * (i & 7);
      v[q][j] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < job.R && n < job.N) {
        const float* sp = job.src + (size_t)r * job.N + n;
        if (vec_ok && n + 3 < job.N) v[q][j] = *reinterpret_cast<const float4*>(sp);
        else { v[q][j].x = sp[0]; if (n + 1 < job.N) v[q][j].y = sp[1]; if (n + 2 < job.N) v[q][j].z = sp[2]; if (n + 3 < job.N) v[q][j].w = sp[3]; }
      }
    }
#pragma unroll
  for (int q = 0; q < P2_SUB; ++q)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int i = tid + 256 * j, rr = i >> 3, c4 = i & 7, r = r0 + rr, n = nb + 32 * q + 4 * c4;
      if (job.transpose) {
        tile[q][rr][4 * c4] = v[q][j].x; tile[q][rr][4 * c4 + 1] = v[q][j].y; tile[q][rr][4 * c4 + 2] = v[q][j].z; tile[q][rr][4 * c4 + 3] = v[q][j].w;
      } else if (r < job.R && n < job.N) {      // natural layout: dst[r * ld + off0 + n], 8-byte runs of 4
        const float x[4] = {v[q][j].x, v[q][j].y, v[q][j].z, v[q][j].w};
        uint16_t p[3][4];
#pragma unroll
        for (int u = 0; u < 4; ++u) split3(x[u], p[0][u], p[1][u], p[2][u]);
#pragma unroll
        for (int k = 0; k < 3; ++k) {          // (a constant trip count keeps p[] and job.dst[] in registers)
          if (k == job.np) break;
          uint16_t* d = job.dst[k] + (size_t)r * job.ld + job.off0 + n;
          if (n + 3 < job.N && (((size_t)r * job.ld + job.off0 + n) & 3) == 0)
            *reinterpret_cast<uint2*>(d) = make_uint2((uint32_t)p[k][0] | ((uint32_t)p[k][1] << 16), (uint32_t)p[k][2] | ((uint32_t)p[k][3] << 16));
          else
            for (int u = 0; u < 4; ++u) if (n + u < job.N) d[u] = p[k][u];
        }
      }
    }
  if (!job.transpose) return;
  __syncthreads();
  // ---- transposed copy: dst[(n + off0) * ld + r]; thread = (n, group of 8 r) of every sub-tile
  const int nn = tid >> 3, g8 = tid & 7, rb = r0 + 8 * g8;
#pragma unroll
  for (int q = 0; q < P2_SUB; ++q) {
    const int n = nb + 32 * q + nn;
    if (n < job.N && rb < job.R) {
      uint16_t p[3][8];
#pragma unroll
      for (int u = 0; u < 8; ++u) split3(tile[q][8 * g8 + u][nn], p[0][u], p[1][u], p[2][u]);
      const size_t o = (size_t)(n + job.off0) * job.ld + rb;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        if (k == job.np) break;
        uint16_t* d = job.dst[k] + o;
        if (job.k1_ci) {
          for (int u = 0; u < 8; ++u) if (rb + u < job.R) d[conv1_krow(rb + u, job.k1_ci) - rb] = p[k][u];
        } else if (rb + 7 < job.R && (o & 7) == 0)
          *reinterpret_cast<uint4*>(d) = make_uint4((uint32_t)p[k][0] | ((uint32_t)p[k][1] << 16), (uint32_t)p[k][2] | ((uint32_t)p[k][3] << 16),
                                                    (uint32_t)p[k][4] | ((uint32_t)p[k][5] << 16), (uint32_t)p[k][6] | ((uint32_t)p[k][7] << 16));
        else
          for (int u = 0; u < 8; ++u) if (rb + u < job.R) d[u] = p[k][u];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host helpers
// ONE map over the np equidistant planes of a tensor: the given geometry plus an outermost plane dimension.  The box covers all
// planes (one instruction fetches them, stacked plane after plane in shared memory) when one plane's box is a whole number of
// 1024-byte swizzle atoms, else one plane (an instruction per plane, plane = last coordinate).  Distinct maps per plane cost a
// descriptor fetch per instruction, whatever the box size.  Returns the map index or -1.
int add_maps(V2State& v, uint16_t* const* planes, int np, int rank, std::initializer_list<uint64_t> dims, std::initializer_list<uint64_t> strides_b,
             std::initializer_list<uint32_t> box, std::initializer_list<uint32_t> estr = {}, bool allow_whole = true, int swizzle = 128) {
  uint64_t d[5] = {1, 1, 1, 1, 1}, s[5] = {0, 0, 0, 0, 0};
  uint32_t bx[5] = {1, 1, 1, 1, 1}, es[5] = {1, 1, 1, 1, 1};
  int i = 0; for (auto x : dims) d[i++] = x;
  i = 0; for (auto x : strides_b) s[i++] = x;
  i = 0; for (auto x : box) bx[i++] = x;
  i = 0; for (auto x : estr) es[i++] = x;
  if (rank >= 5 || np < 1) return -1;
  size_t rows = 1;
  for (int k = 1; k < rank; ++k) rows *= (bx[k] + es[k] - 1) / es[k];
  const size_t box_bytes = rows * bx[0] * 2;
  const bool whole = allow_whole && np > 1 && box_bytes % 1024 == 0;
  const long long pitch = np > 1 ? (long long)((const char*)planes[1] - (const char*)planes[0]) : 16;
  for (int p = 2; p < np; ++p)
    if ((const char*)planes[p] - (const char*)planes[p - 1] != pitch) return -1;
  if (pitch <= 0 || pitch % 16) return -1;
  d[rank] = (uint64_t)np; s[rank - 1] = (uint64_t)pitch; bx[rank] = whole ? (uint32_t)np : 1u; es[rank] = 1;
  CUtensorMap m;
  if (cg_encode_map(&m, planes[0], rank + 1, d, s, bx, es, swizzle) != 0) return -1;
  v.maps.push_back(m);
  v.map_whole.push_back(whole ? 1 : 0);
  v.map_box_bytes.push_back((int)box_bytes);
  return (int)v.maps.size() - 1;
}

const V2State* g_mk_state = nullptr;     // set by v2_create: mk_load looks up whether the map's box holds every plane
CgLoad mk_load(int map, int rank, int smem_off) {
  CgLoad L;
  memset(&L, 0, sizeof(L));
  L.map = map; L.rank = rank + 1; L.smem_off = smem_off;        // + the plane dimension
  L.plane_box = g_mk_state->map_whole[map];
  L.box_bytes = g_mk_state->map_box_bytes[map];
  return L;
}

// K-major problem skeleton: A tile 128 rows x 64 k, B tile N rows x 64 k, `planes` BF16 planes
CgProblem kmajor(int planes, int n_tile, int chunks, int n2, int a_box_rows) {
  CgProblem P;
  memset(&P, 0, sizeof(P));
  P.tiles_m = P.tiles_n = P.splits = 1;
  P.chunks = chunks; P.n2 = n2;
  P.planes = planes;
  P.a_off = 0; P.a_pstride = 128 * 128;
  P.b_off = planes * P.a_pstride; P.b_pstride = n_tile * 128;
  P.tx_bytes = planes * (a_box_rows * 128 + n_tile * 128);
  P.mn_major = 0; P.ksteps = 4; P.a_kstep = P.b_kstep = 32; P.a_kstep2 = 64;
  P.a_desc = P.b_desc = cg_desc_bits(128, false, 0); P.a_moff = 64 * 128;
  P.umma_n = n_tile;
  P.nprod = planes == 3 ? 6 : (planes == 2 ? 3 : 1);
  P.d0 = 1 << 20; P.d1 = 1;
  P.grp_stride = 32; P.f_grp = 32; P.bias_grp = 32;
  P.scale = 1.f;
  return P;
}

// MN-major (wgrad) problem skeleton: rows = reduction index (kr rows per chunk), A = a_atoms x (64 m x kr), B = b_atoms x (64 n x kr)
CgProblem mnmajor(int planes, int kr, int a_atoms, int b_atoms, int chunks) {
  CgProblem P;
  memset(&P, 0, sizeof(P));
  P.tiles_m = P.tiles_n = P.splits = 1;
  P.chunks = chunks; P.n2 = chunks > 0 ? chunks : 1;
  P.planes = planes;
  const int atom = kr * 128;
  // A region: [atom 0: plane 0, plane 1, ..][atom 1: ..] (each atom is one box with the planes stacked; M = 128 = two atoms);
  // B region: [plane 0: atoms][plane 1: atoms] so that [B_0 | B_1] is one wide operand
  P.a_off = 0; P.a_pstride = atom;
  P.b_off = 2 * planes * atom; P.b_pstride = b_atoms * atom;
  P.tx_bytes = planes * (a_atoms + b_atoms) * atom;
  P.mn_major = 1; P.ksteps = kr / 16; P.a_kstep = P.b_kstep = 2048; P.a_kstep2 = 4096;
  P.a_lbo = planes * atom; P.b_lbo = atom;
  P.a_desc = cg_desc_bits(128, true, P.a_lbo); P.b_desc = cg_desc_bits(128, true, P.b_lbo); P.a_moff = P.a_lbo;
  P.umma_n = 64 * b_atoms;
  P.nprod = planes == 3 ? 6 : (planes == 2 ? 3 : 1);
  P.d0 = 1 << 20; P.d1 = 1;
  P.grp_stride = 32; P.f_grp = 32; P.bias_grp = 32;
  P.scale = 1.f;
  P.epi = CG_EPI_WGRAD; P.rows_tile = 128;
  return P;
}

int push_group(b2g_sac* h, std::vector<CgGroup>& list, CgGroup& g, const char* name) {
  g.name = name;
  if (cg_finalize(g, cg_smem_limit()) != 0) return b2g_fail(B2G_EINVAL, std::string("engine v2: stage ring of group ") + name + " does not fit shared memory");
  for (int i = 0; i < g.n; ++i) {
    const CgProblem& P = g.host[i];
    if (P.planes * P.umma_n > 256) return b2g_fail(B2G_EINVAL, std::string("engine v2: planes x tile width exceeds one accumulator buffer (group ") + name + ")");
    if (!cg_shape_supported(P.umma_n, P.nprod, P.mn_major != 0, P.ksteps))
      return b2g_fail(B2G_EINVAL, std::string("engine v2: no cg_kernel instance for the tile shape of a problem in group ") + name);
    if (P.tm_sub > 1 && !cg_epi_handoff(P.epi))     // only the epilogue warpgroup maps bands (cg.cuh: tm_sub)
      return b2g_fail(B2G_EINVAL, std::string("engine v2: a banded problem must have an ACT or DGRAD epilogue (group ") + name + ")");
    g.flops += 2.0 * P.tiles_m * 128.0 * P.tiles_n * P.umma_n * P.chunks * 64.0;      // issued (tile-padded) work
  }
  list.push_back(g);
  return 0;
}

// Concatenates layer groups into one launch and chains them by arrival counters.  A wire says: problem `ci` of part `cons` reads
// rows [x * dep_rows, (x + 1) * dep_rows) of the output of problem `pi` of part `prod`, x = its row-tile index (by_chunk = 0) or its
// K-chunk index (by_chunk = 1: weight gradients reduce over the producer's rows); the producer finishes dep_rows_tile such rows per tile.
struct Wire { int cons, ci, prod, pi, dep_rows, dep_rows_tile, by_chunk; };
int fuse_groups(b2g_sac* h, const std::vector<const CgGroup*>& parts, const std::vector<Wire>& wires, const char* name, std::vector<CgGroup>& out, int& n_ctr) {
  CgGroup f;
  std::vector<int> first(parts.size());
  for (size_t gi = 0; gi < parts.size(); ++gi) {
    first[gi] = f.n;
    for (int i = 0; i < parts[gi]->n; ++i) {
      if (f.n >= CG_MAX_PROBLEMS) return b2g_fail(B2G_EINVAL, std::string("engine v2: too many problems in fused launch ") + name);
      f.host[f.n++] = parts[gi]->host[i];
    }
  }
  std::vector<int> ctr_of(f.n, -1);
  for (const Wire& w : wires) {
    const int pi = first[w.prod] + w.pi, qi = first[w.cons] + w.ci;
    CgProblem& Pp = f.host[pi];
    CgProblem& Pc = f.host[qi];
    if (!cg_epi_handoff(Pp.epi))       // only the epilogue warpgroup signals finished tiles (cg.cuh: cg_epi_handoff)
      return b2g_fail(B2G_EINVAL, std::string("engine v2: a wired producer must have an ACT or DGRAD epilogue (fused launch ") + name + ")");
    if (Pc.dep_ctr && ctr_of[pi] < 0) {
      // a second producer of the same consumer (the two nets' conv2 dgrads both write dZ1): it signals the first one's counters
      ctr_of[pi] = (int)(intptr_t)Pc.dep_ctr - 1;
      Pc.dep_expect += Pp.ws ? Pp.tiles_n : Pp.tiles_n * Pp.splits;
      continue;
    }
    // a split-K producer signals its counters from the tiles of every split (or, finalised, from the last arriver): a split
    // without chunks skips its tile and would leave the counters short forever
    if (Pp.splits > 1 && (Pp.splits - 1) * ((Pp.chunks + Pp.splits - 1) / Pp.splits) >= Pp.chunks)
      return b2g_fail(B2G_EINVAL, std::string("engine v2: a wired split-K producer has an empty split (fused launch ") + name + ")");
    if (ctr_of[pi] < 0) { ctr_of[pi] = n_ctr; n_ctr += Pp.tiles_m; }
    Pc.dep_rows = w.dep_rows; Pc.dep_rows_tile = w.dep_rows_tile; Pc.dep_tiles = Pp.tiles_m; Pc.dep_by_chunk = w.by_chunk;
    Pc.dep_expect = Pp.ws ? Pp.tiles_n : Pp.tiles_n * Pp.splits;   // x the signalling epilogue warps per tile (kernel side); split-K
                                                                   // tiles with finalisation are signalled by their last arriver only
    Pc.dep_ctr = (const int*)(intptr_t)(ctr_of[pi] + 1);        // counter index + 1; turned into pointers once the array exists
  }
  for (int i = 0; i < f.n; ++i) f.host[i].done_ctr = (int*)(intptr_t)(ctr_of[i] + 1);
  return push_group(h, out, f, name);
}

void bind_counters(std::vector<CgGroup>& groups, int* base) {
  for (CgGroup& g : groups)
    for (int i = 0; i < g.n; ++i) {
      CgProblem& P = g.host[i];
      const intptr_t d = (intptr_t)P.done_ctr, c = (intptr_t)P.dep_ctr;
      P.done_ctr = d ? base + (d - 1) : nullptr;
      P.dep_ctr = c ? base + (c - 1) : nullptr;
    }
}

// A K-split of `chunks` chunks into `splits` takes ceil(chunks / splits) chunks per split, so some counts leave the last
// splits with none (16 chunks in 5 splits: 4 + 4 + 4 + 4 + 0).  An empty split of a finalised split-K tile never arrives at
// the tile's ws_cnt, so no split is the last arriver, the tile is never finished and the tiles that wait on it spin forever.
// Such a count is refused at create, with the counts that do work in the message.
int check_split(const char* var, int chunks, int splits) {
  auto empty = [chunks](int s) { return (s - 1) * ((chunks + s - 1) / s) >= chunks; };
  if (!empty(splits)) return 0;
  std::string ok;
  for (int s = 1; s <= chunks; ++s)
    if (!empty(s)) ok += (ok.empty() ? "" : ", ") + std::to_string(s);
  return b2g_fail(B2G_EINVAL, std::string(var) + "=" + std::to_string(splits) + " leaves a K-split of " + std::to_string(chunks) +
                                  " chunks empty; use one of " + ok);
}

}  // namespace

// ================================================================================================ create
int v2_alloc(b2g_sac* h) {
  V2State& v = h->v2;
  const int B = h->B, Cp = s2d_channels(h->Cimg), K1 = 64 * Cp, KF = v.KF;
  const size_t n1 = (size_t)B * 225 * 32, n2 = (size_t)B * 36 * 64, n3 = (size_t)B * 1024, ns = (size_t)B * 4096 * Cp, nf = (size_t)B * KF;
  // ---- activations: one block per layer, [net][plane] with uniform strides (conv1 writes two nets from one tile)
  uint16_t *bH1, *bH2, *bH3, *bF, *bS;
  if (int rc = dev_alloc(h->allocs, h->stream, &bH1, 9 * n1)) return rc;
  if (int rc = dev_alloc(h->allocs, h->stream, &bH2, 9 * n2)) return rc;
  if (int rc = dev_alloc(h->allocs, h->stream, &bH3, 9 * n3)) return rc;
  if (int rc = dev_alloc(h->allocs, h->stream, &bF, 9 * nf)) return rc;
  if (int rc = dev_alloc(h->allocs, h->stream, &bS, 6 * ns)) return rc;
  for (int n = 0; n < 3; ++n)
    for (int p = 0; p < 3; ++p) {
      v.H1[n][p] = bH1 + (n * 3 + p) * n1; v.H2[n][p] = bH2 + (n * 3 + p) * n2; v.H3[n][p] = bH3 + (n * 3 + p) * n3;
      v.F[n][p] = bF + (n * 3 + p) * nf;
    }
  for (int w = 0; w < 2; ++w) for (int p = 0; p < 3; ++p) v.S[w][p] = bS + (w * 3 + p) * ns;
  if (int rc = dev_alloc(h->allocs, h->stream, &v.z0v, (size_t)B * 3 * h->H)) return rc;
  // ---- gradient maps (2 planes) and natural-layout weight planes of the backward chain.  The planes of a tensor are
  //      equidistant in one allocation: the tensor maps address them through an extra (outermost) plane dimension
  auto palloc = [&](uint16_t** arr, int np, size_t count) -> int {
    const size_t pitch = (count + 63) / 64 * 64;
    uint16_t* base = nullptr;
    if (int rc = dev_alloc(h->allocs, h->stream, &base, pitch * np)) return rc;
    for (int p = 0; p < np; ++p) arr[p] = base + p * pitch;
    return 0;
  };
  if (int rc = palloc(v.dz0pi, 2, (size_t)B * h->H)) return rc;
  if (int rc = palloc(v.dz0v, 2, (size_t)B * 3 * h->H)) return rc;
  if (int rc = palloc(v.dZ1, 2, (size_t)B * 225 * 64)) return rc;
  for (int n = 0; n < 2; ++n) {
    if (int rc = palloc(v.dZ4[n], 2, (size_t)B * 512)) return rc;
    if (int rc = palloc(v.dZ3[n], 2, n3)) return rc;
    if (int rc = palloc(v.dZ2[n], 2, n2)) return rc;
    if (int rc = palloc(v.W2n[n], 2, 512 * 64)) return rc;
    if (int rc = palloc(v.W3n[n], 2, 576 * 64)) return rc;
    if (int rc = palloc(v.Wfn[n], 2, 1024 * 512)) return rc;
    if (int rc = palloc(v.K0n[n], 2, (size_t)KF * (n == 1 ? 3 : 1) * h->H)) return rc;
  }
  // ---- weight planes
  if (int rc = palloc(v.W1T[0], 3, (size_t)64 * K1)) return rc;
  if (int rc = palloc(v.W1T[1], 3, (size_t)32 * K1)) return rc;
  for (int n = 0; n < 3; ++n) {
    if (int rc = palloc(v.W2T[n], 3, 64 * 512)) return rc;
    if (int rc = palloc(v.W3T[n], 3, 64 * 576)) return rc;
    if (int rc = palloc(v.WfT[n], 3, 512 * 1024)) return rc;
    if (int rc = palloc(v.K0T[n], 3, (size_t)(n == 1 ? 3 : 1) * h->H * KF)) return rc;
  }
  return 0;
}

int v2_create(b2g_sac* h) {
  V2State& v = h->v2;
  g_mk_state = &v;
  const int B = h->B, Ci = h->Cimg, Cp = s2d_channels(Ci), K1 = 64 * Cp, KF = v.KF, FS = h->FS, H = h->H;
  const size_t n1 = (size_t)B * 225 * 32;
  // ---- plane jobs (weights change every step)
  const char* nets[3] = {"model/pi", "model/values_fn", "target/values_fn"};
  std::vector<Plane2Job> jobs;
  int start = 0;
  auto add_job = [&](const float* src, int R, int N, uint16_t* const* dst, int np, int transpose, int ld, int off0) {
    Plane2Job j{};
    j.src = src; j.R = R; j.N = N; j.np = np; j.transpose = transpose; j.ld = ld; j.off0 = off0; j.tile_start = start;
    for (int k = 0; k < np; ++k) j.dst[k] = dst[k];
    start += ((R + 63) / 64) * ((N + 32 * P2_SUB - 1) / (32 * P2_SUB));
    jobs.push_back(j);
  };
  add_job(h->p(h->cnn_t("model/pi", 0, "w")), 64 * Ci, 32, v.W1T[0], 3, 1, K1, 0);
  jobs.back().k1_ci = Ci;
  add_job(h->p(h->cnn_t("model/values_fn", 0, "w")), 64 * Ci, 32, v.W1T[0], 3, 1, K1, 32);
  jobs.back().k1_ci = Ci;
  add_job(h->p(h->cnn_t("target/values_fn", 0, "w")), 64 * Ci, 32, v.W1T[1], 3, 1, K1, 0);
  jobs.back().k1_ci = Ci;
  for (int n = 0; n < 3; ++n) {
    add_job(h->p(h->cnn_t(nets[n], 1, "w")), 512, 64, v.W2T[n], 3, 1, 512, 0);
    add_job(h->p(h->cnn_t(nets[n], 2, "w")), 576, 64, v.W3T[n], 3, 1, 576, 0);
    add_job(h->p(h->cnn_t(nets[n], 3, "w")), 1024, 512, v.WfT[n], 3, 1, 1024, 0);
  }
  add_job(h->p("model/pi/fc0/kernel"), h->feat_dim, H, v.K0T[0], 3, 1, KF, 0);
  add_job(h->p("model/values_fn/vf/fc0/kernel"), h->feat_dim, H, v.K0T[1], 3, 1, KF, 0);
  add_job(h->p("model/values_fn/qf1/fc0/kernel"), h->feat_dim + h->A, H, v.K0T[1], 3, 1, KF, H);
  add_job(h->p("model/values_fn/qf2/fc0/kernel"), h->feat_dim + h->A, H, v.K0T[1], 3, 1, KF, 2 * H);
  add_job(h->p("target/values_fn/vf/fc0/kernel"), h->feat_dim, H, v.K0T[2], 3, 1, KF, 0);
  v.plane_ctas_fwd = start;      // the forward-layout jobs above, then the backward layouts (first read by bwd_fused)
  for (int n = 0; n < 2; ++n) {
    add_job(h->p(h->cnn_t(nets[n], 1, "w")), 512, 64, v.W2n[n], 2, 0, 64, 0);
    add_job(h->p(h->cnn_t(nets[n], 2, "w")), 576, 64, v.W3n[n], 2, 0, 64, 0);
    add_job(h->p(h->cnn_t(nets[n], 3, "w")), 1024, 512, v.Wfn[n], 2, 0, 512, 0);
  }
  add_job(h->p("model/pi/fc0/kernel"), h->feat_dim, H, v.K0n[0], 2, 0, H, 0);
  add_job(h->p("model/values_fn/vf/fc0/kernel"), h->feat_dim, H, v.K0n[1], 2, 0, 3 * H, 0);
  add_job(h->p("model/values_fn/qf1/fc0/kernel"), h->feat_dim + h->A, H, v.K0n[1], 2, 0, 3 * H, H);
  add_job(h->p("model/values_fn/qf2/fc0/kernel"), h->feat_dim + h->A, H, v.K0n[1], 2, 0, 3 * H, 2 * H);
  v.n_plane_jobs = (int)jobs.size();
  v.plane_ctas = start;
  Plane2Job* dj = nullptr;
  if (int rc = dev_alloc(h->allocs, h->stream, &dj, jobs.size())) return rc;
  CK(cudaMemcpyAsync(dj, jobs.data(), jobs.size() * sizeof(Plane2Job), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  v.plane_jobs = dj;
  {
    std::vector<int> cj((size_t)start);
    for (size_t k = 0; k < jobs.size(); ++k)
      for (int t = jobs[k].tile_start; t < (k + 1 < jobs.size() ? jobs[k + 1].tile_start : start); ++t) cj[t] = (int)k;
    if (int rc = upload_table(h->allocs, h->stream, cj, &v.plane_cta_job)) return rc;
  }

  { const char* e = getenv("B2G_SPLIT_FC1"); v.split_fc1 = e ? std::max(1, atoi(e)) : 3; }
  { const char* e = getenv("B2G_SPLIT_FC1_DGRAD"); v.split_fc1_dgrad = e ? std::max(1, atoi(e)) : 1; }
  // ================================================================================ forward problems (6-product mode)
  const int NP = 3;
  const long long h1_net = (long long)3 * n1;       // element distance between the same plane of consecutive nets
  // ---- conv1: [obs -> pi | vf] (N = 64, two output tensors) and [next_obs -> target] (N = 32), a 2x2 stride-1 convolution over S.
  //      The sample is folded into the block row (monotonic strides): row tile tm = 2 s + t (output rows oy 8t .. 8t + 7, ox 0 .. 15 of
  //      sample s) reads block rows 8 tm + a.  Block row 16 s + 16 belongs to the next sample (the last sample's is out of bounds);
  //      like X = 15 + 1 it only reaches the junk rows ox = 15 and oy = 15, which the epilogue does not store.
  //      Cp = 4: S as {64, 16 X, 16 B Y}; K-chunk = window (c1, c2) = (a, a'), the box {64, 16, 8} at (0, a', 8 tm + a).
  //      Cp = 1: S as {32, 15 X, 16 B Y} with a 32-byte X stride, so that a row holds blocks X and X + 1 = windows (a, 0) and (a, 1)
  //      (the view overlaps itself along X, like conv2's); the box {32, 16, 8} at (0, 0, 8 tm + a) holds k-steps 2a and 2a + 1
  //      (64-byte rows, X = 15 out of bounds), one K-chunk of two such boxes.
  {
    CgGroup g;
    for (int w = 0; w < 2; ++w) {
      const int N = w == 0 ? 64 : 32;
      const int mA = Cp == 1 ? add_maps(v, v.S[w], NP, 3, {32, 15, (uint64_t)B * 16}, {32, 512}, {32, 16, 8}, {}, true, 64)
                             : add_maps(v, v.S[w], NP, 3, {64, 16, (uint64_t)B * 16}, {128, 2048}, {64, 16, 8});
      const int mB = add_maps(v, v.W1T[w], NP, 2, {(uint64_t)K1, (uint64_t)N}, {(uint64_t)K1 * 2}, {64, (uint32_t)N});
      if (mA < 0 || mB < 0) return b2g_fail(B2G_ECUDA, "engine v2: cuTensorMapEncodeTiled failed (conv1)");
      CgProblem P;
      if (Cp == 1) {
        // k-step 2a + a' = box a, bytes [32 a', 32 a' + 32) of its 64-byte rows
        P = kmajor(NP, N, 1, 1, 128);
        P.a_pstride = 128 * 64; P.a_kstep = 32; P.a_kstep2 = NP * P.a_pstride;
        P.b_off = 2 * P.a_kstep2;
        P.tx_bytes = NP * (2 * 128 * 64 + N * 128);
        P.a_desc = cg_desc_bits(64, false, 0); P.a_moff = 64 * 64;
        P.nloads = 3;
        for (int a = 0; a < 2; ++a) { P.ld[a] = mk_load(mA, 3, a * P.a_kstep2); P.ld[a].c0[2] = a; P.ld[a].d_tm[2] = 8; }
        P.ld[2] = mk_load(mB, 2, P.b_off);
      } else {
        P = kmajor(NP, N, 4, 2, 128);
        P.nloads = 2;
        P.ld[0] = mk_load(mA, 3, 0); P.ld[0].d_tm[2] = 8; P.ld[0].d_c1[2] = 1; P.ld[0].d_c2[1] = 1;
        P.ld[1] = mk_load(mB, 2, P.b_off); P.ld[1].d_c1[0] = 128; P.ld[1].d_c2[0] = 64;
      }
      P.tiles_m = 2 * B;
      P.epi = CG_EPI_ACT; P.rows_tile = 128; P.lim_rows = 2 * B * 128;
      P.d0 = 16; P.d1 = 8; P.o0 = 32; P.o1 = 15 * 32; P.o_tm = 225 * 32;      // row (oy - 8t, ox) of band t of sample s
      P.tm_sub = 2; P.o_sub = 8 * 15 * 32; P.lim_i0 = 15; P.lim_i1 = 15;
      P.n_valid = N; P.out_planes = 3;
      P.grp_stride = (int)h1_net;
      const int net0 = w == 0 ? 0 : 2;
      for (int p = 0; p < 3; ++p) P.out_p[p] = v.H1[net0][p];
      P.bias = h->p(h->cnn_t(nets[net0], 0, "b"));
      P.bias_grp = w == 0 ? (int)(h->p(h->cnn_t("model/values_fn", 0, "b")) - h->p(h->cnn_t("model/pi", 0, "b"))) : 32;
      g.host[g.n++] = P;
    }
    if (int rc = push_group(h, v.fwd, g, "conv1_fwd")) return rc;
  }
  // ---- conv2: 4x4 stride-2 patches of H1 as a 4-D view {2 pixels x 32 ch, x, y, b} with element strides {1,2,2,1}
  {
    CgGroup g;
    for (int n = 0; n < 3; ++n) {
      const int mA = add_maps(v, v.H1[n], NP, 4, {64, 14, 15, (uint64_t)B}, {64, 15 * 64, 225 * 64}, {64, 12, 12, 3}, {1, 2, 2, 1});
      const int mB = add_maps(v, v.W2T[n], NP, 2, {512, 64}, {1024}, {64, 64});
      if (mA < 0 || mB < 0) return b2g_fail(B2G_ECUDA, "engine v2: cuTensorMapEncodeTiled failed (conv2)");
      CgProblem P = kmajor(NP, 64, 8, 2, 108);
      P.nloads = 2;
      P.ld[0] = mk_load(mA, 4, 0); P.ld[0].d_tm[3] = 3; P.ld[0].d_c1[2] = 1; P.ld[0].d_c2[1] = 2;
      P.ld[1] = mk_load(mB, 2, P.b_off); P.ld[1].d_c1[0] = 128; P.ld[1].d_c2[0] = 64;
      P.tiles_m = (B + 2) / 3;
      P.epi = CG_EPI_ACT; P.rows_tile = 108; P.lim_rows = B * 36;
      P.o_tm = 108 * 64; P.o0 = 64; P.n_valid = 64; P.out_planes = 3;
      for (int p = 0; p < 3; ++p) P.out_p[p] = v.H2[n][p];
      P.bias = h->p(h->cnn_t(nets[n], 1, "b")); P.bias_grp = 32;
      g.host[g.n++] = P;
    }
    if (int rc = push_group(h, v.fwd, g, "conv2_fwd")) return rc;
  }
  // ---- conv3: 3x3 stride-1 windows of H2, 8 samples (128 rows) per tile
  {
    CgGroup g;
    for (int n = 0; n < 3; ++n) {
      const int mA = add_maps(v, v.H2[n], NP, 4, {64, 6, 6, (uint64_t)B}, {128, 6 * 128, 36 * 128}, {64, 4, 4, 8});
      const int mB = add_maps(v, v.W3T[n], NP, 2, {576, 64}, {1152}, {64, 64});
      if (mA < 0 || mB < 0) return b2g_fail(B2G_ECUDA, "engine v2: cuTensorMapEncodeTiled failed (conv3)");
      CgProblem P = kmajor(NP, 64, 9, 3, 128);
      P.nloads = 2;
      P.ld[0] = mk_load(mA, 4, 0); P.ld[0].d_tm[3] = 8; P.ld[0].d_c1[2] = 1; P.ld[0].d_c2[1] = 1;
      P.ld[1] = mk_load(mB, 2, P.b_off); P.ld[1].d_c1[0] = 192; P.ld[1].d_c2[0] = 64;
      P.tiles_m = (B + 7) / 8;
      P.epi = CG_EPI_ACT; P.rows_tile = 128; P.lim_rows = B * 16;
      P.o_tm = 128 * 64; P.o0 = 64; P.n_valid = 64; P.out_planes = 3;
      for (int p = 0; p < 3; ++p) P.out_p[p] = v.H3[n][p];
      P.bias = h->p(h->cnn_t(nets[n], 2, "b")); P.bias_grp = 32;
      g.host[g.n++] = P;
    }
    if (int rc = push_group(h, v.fwd, g, "conv3_fwd")) return rc;
  }
  // ---- cnn_fc1: [B,1024] x [1024,512] -> feature rows (planes + the fp32 copy the head kernels read)
  {
    CgGroup g;
    for (int n = 0; n < 3; ++n) {
      const int mA = add_maps(v, v.H3[n], NP, 2, {1024, (uint64_t)B}, {2048}, {64, 128});
      const int mB = add_maps(v, v.WfT[n], NP, 2, {1024, 512}, {2048}, {64, 64});
      if (mA < 0 || mB < 0) return b2g_fail(B2G_ECUDA, "engine v2: cuTensorMapEncodeTiled failed (cnn_fc1)");
      CgProblem P = kmajor(NP, 64, 16, 16, 128);
      P.nloads = 2;
      P.ld[0] = mk_load(mA, 2, 0); P.ld[0].d_tm[1] = 128; P.ld[0].d_c2[0] = 64;
      P.ld[1] = mk_load(mB, 2, P.b_off); P.ld[1].d_tn[1] = 64; P.ld[1].d_c2[0] = 64;
      P.tiles_m = (B + 127) / 128; P.tiles_n = 8;
      P.epi = CG_EPI_ACT; P.rows_tile = 128; P.lim_rows = B;
      P.o_tm = (long long)128 * KF; P.o0 = KF; P.n_valid = 512; P.out_planes = 3;
      for (int p = 0; p < 3; ++p) P.out_p[p] = v.F[n][p];
      P.bias = h->p(h->cnn_t(nets[n], 3, "b")); P.bias_grp = 32;
      P.out_f = h->F[n]; P.f_tm = (long long)128 * FS; P.f0 = FS; P.f_grp = 32;
      if (v.split_fc1 > 1) {
        // 48 tiles of 16 K-chunks would hold 48 of the 132 SMs for the longest stretch of the forward launch: three K-splits per
        // tile, fp32 partial sums in a workspace, the last split to arrive finishes the tile (cg.cuh: ws)
        P.splits = v.split_fc1;
        if (int rc = check_split("B2G_SPLIT_FC1", P.chunks, P.splits)) return rc;
        if (int rc = dev_alloc(h->allocs, h->stream, &P.ws, (size_t)P.tiles_m * P.tiles_n * 128 * 64)) return rc;
        if (int rc = dev_alloc(h->allocs, h->stream, &P.ws_cnt, (size_t)P.tiles_m * P.tiles_n * CG_EPI_WARPS)) return rc;
      }
      g.host[g.n++] = P;
    }
    if (int rc = push_group(h, v.fwd, g, "fc1_fwd")) return rc;
  }
  // ---- head fc0 layers: pi [513->H], values vf|q1|q2 [518->3H] on the shared feature rows, target vf
  {
    CgGroup g;
    float* z0out[3] = {h->z0[0], v.z0v, h->z0[4]};
    for (int n = 0; n < 3; ++n) {
      const int Nn = n == 1 ? 3 * H : H;
      const int mA = add_maps(v, v.F[n], NP, 2, {(uint64_t)KF, (uint64_t)B}, {(uint64_t)KF * 2}, {64, 128});
      const int mB = add_maps(v, v.K0T[n], NP, 2, {(uint64_t)KF, (uint64_t)Nn}, {(uint64_t)KF * 2}, {64, 64});
      if (mA < 0 || mB < 0) return b2g_fail(B2G_ECUDA, "engine v2: cuTensorMapEncodeTiled failed (fc0)");
      CgProblem P = kmajor(NP, 64, KF / 64, KF / 64, 128);
      P.nloads = 2;
      P.ld[0] = mk_load(mA, 2, 0); P.ld[0].d_tm[1] = 128; P.ld[0].d_c2[0] = 64;
      P.ld[1] = mk_load(mB, 2, P.b_off); P.ld[1].d_tn[1] = 64; P.ld[1].d_c2[0] = 64;
      P.tiles_m = (B + 127) / 128; P.tiles_n = Nn / 64;
      P.epi = CG_EPI_RAW; P.rows_tile = 128; P.lim_rows = B;
      P.o_tm = (long long)128 * Nn; P.o0 = Nn; P.n_valid = Nn;
      P.splits = P.chunks; P.atomic = 1;      // one K-chunk per CTA, fp32 red.add into the zeroed z0 block (10 serial 9-chunk tiles otherwise)
      P.out_f = z0out[n];
      g.host[g.n++] = P;
    }
    if (int rc = push_group(h, v.fwd, g, "heads_fc0")) return rc;
  }

  // ================================================================================ backward problems (3-product mode)
  const int NB = 2;
  // ---- heads dgrad: dZ4 = dz0 . K0^T, masked by the cnn_fc1 ReLU (F > 0)
  {
    CgGroup g;
    for (int n = 0; n < 2; ++n) {
      const int Kd = n == 0 ? H : 3 * H;
      uint16_t* const* dz = n == 0 ? v.dz0pi : v.dz0v;
      const int mA = add_maps(v, dz, NB, 2, {(uint64_t)Kd, (uint64_t)B}, {(uint64_t)Kd * 2}, {64, 128});
      const int mB = add_maps(v, v.K0n[n], NB, 2, {(uint64_t)Kd, (uint64_t)KF}, {(uint64_t)Kd * 2}, {64, 128});
      if (mA < 0 || mB < 0) return b2g_fail(B2G_ECUDA, "engine v2: cuTensorMapEncodeTiled failed (heads dgrad)");
      CgProblem P = kmajor(NB, 128, Kd / 64, Kd / 64, 128);
      P.nloads = 2;
      P.ld[0] = mk_load(mA, 2, 0); P.ld[0].d_tm[1] = 128; P.ld[0].d_c2[0] = 64;
      P.ld[1] = mk_load(mB, 2, P.b_off); P.ld[1].d_tn[1] = 128; P.ld[1].d_c2[0] = 64;
      P.tiles_m = (B + 127) / 128; P.tiles_n = 4;
      P.epi = CG_EPI_DGRAD; P.rows_tile = 128; P.lim_rows = B;
      P.o_tm = 128 * 512; P.o0 = 512; P.n_valid = 512; P.out_planes = 2;
      for (int p = 0; p < 2; ++p) P.out_p[p] = v.dZ4[n][p];
      P.mask = v.F[n][0]; P.m_tm = (long long)128 * KF; P.m0 = KF;
      P.colsum = h->g(h->cnn_t(nets[n], 3, "b")); P.colsum_mask = 511;
      g.host[g.n++] = P;
    }
    if (int rc = push_group(h, v.bwd_groups, g, "heads_dgrad")) return rc;
  }
  // ---- cnn_fc1 backward: dgrad dZ3 = dZ4 . Wf^T (masked by h3 > 0) and wgrad G_Wf = h3^T . dZ4 (MN-major, K = batch)
  {
    CgGroup g;
    for (int n = 0; n < 2; ++n) {
      {
        const int mA = add_maps(v, v.dZ4[n], NB, 2, {512, (uint64_t)B}, {1024}, {64, 128});
        const int mB = add_maps(v, v.Wfn[n], NB, 2, {512, 1024}, {1024}, {64, 128});
        if (mA < 0 || mB < 0) return b2g_fail(B2G_ECUDA, "engine v2: cuTensorMapEncodeTiled failed (fc1 dgrad)");
        CgProblem P = kmajor(NB, 128, 8, 8, 128);
        P.nloads = 2;
        P.ld[0] = mk_load(mA, 2, 0); P.ld[0].d_tm[1] = 128; P.ld[0].d_c2[0] = 64;
        P.ld[1] = mk_load(mB, 2, P.b_off); P.ld[1].d_tn[1] = 128; P.ld[1].d_c2[0] = 64;
        P.tiles_m = (B + 127) / 128; P.tiles_n = 8;
        P.epi = CG_EPI_DGRAD; P.rows_tile = 128; P.lim_rows = B;
        P.o_tm = 128 * 1024; P.o0 = 1024; P.n_valid = 1024; P.out_planes = 2;
        for (int p = 0; p < 2; ++p) P.out_p[p] = v.dZ3[n][p];
        P.mask = v.H3[n][0]; P.m_tm = 128 * 1024; P.m0 = 1024;
        P.colsum = h->g(h->cnn_t(nets[n], 2, "b")); P.colsum_mask = 63;     // dZ3 row = [16 pixels][64 channels]
        if (v.split_fc1_dgrad > 1) {         // 32 tiles of 8 K-chunks at the head of the backward chain: split-K with finalisation
          P.splits = v.split_fc1_dgrad;
          if (int rc = check_split("B2G_SPLIT_FC1_DGRAD", P.chunks, P.splits)) return rc;
          if (int rc = dev_alloc(h->allocs, h->stream, &P.ws, (size_t)P.tiles_m * P.tiles_n * 128 * 128)) return rc;
          if (int rc = dev_alloc(h->allocs, h->stream, &P.ws_cnt, (size_t)P.tiles_m * P.tiles_n * CG_EPI_WARPS)) return rc;
        }
        g.host[g.n++] = P;
      }
      {
        const int mA = add_maps(v, v.H3[n], NB, 2, {1024, (uint64_t)B}, {2048}, {64, 64});
        const int mB = add_maps(v, v.dZ4[n], NB, 2, {512, (uint64_t)B}, {1024}, {64, 64}, {}, false);     // two B atoms per plane
        if (mA < 0 || mB < 0) return b2g_fail(B2G_ECUDA, "engine v2: cuTensorMapEncodeTiled failed (fc1 wgrad)");
        CgProblem P = mnmajor(NB, 64, 2, 2, (B + 63) / 64);
        P.nloads = 4;
        for (int a = 0; a < 2; ++a) {
          P.ld[a] = mk_load(mA, 2, a * P.a_lbo); P.ld[a].c0[0] = 64 * a; P.ld[a].d_tm[0] = 128; P.ld[a].d_c2[1] = 64;
          P.ld[2 + a] = mk_load(mB, 2, P.b_off + a * 8192); P.ld[2 + a].c0[0] = 64 * a; P.ld[2 + a].d_tn[0] = 128; P.ld[2 + a].d_c2[1] = 64;
        }
        P.tiles_m = 8; P.tiles_n = 4;
        P.lim_rows = 1024; P.o_tm = 128 * 512; P.o0 = 512; P.n_valid = 512;
        P.out_f = h->g(h->cnn_t(nets[n], 3, "w")); P.atomic = 0;
        g.host[g.n++] = P;
      }
    }
    if (int rc = push_group(h, v.bwd_groups, g, "fc1_bwd")) return rc;
  }
  // ---- conv3 backward: dgrad over the zero-bordered dZ3 (TMA out-of-bound fill) and wgrad (two kernel positions per M tile)
  {
    CgGroup g;
    std::vector<int> tab(5 * CG_MAX_LOADS * 2, 0);
    for (int tm = 0; tm < 5; ++tm)
      for (int a = 0; a < 2; ++a) {
        const int pos = 2 * tm + a;
        tab[(tm * CG_MAX_LOADS + a) * 2] = pos % 3; tab[(tm * CG_MAX_LOADS + a) * 2 + 1] = pos / 3;
      }
    const int* dtab = nullptr;
    if (int rc = upload_table(h->allocs, h->stream, tab, &dtab)) return rc;
    for (int n = 0; n < 2; ++n) {
      {
        const int mA = add_maps(v, v.dZ3[n], NB, 4, {64, 4, 4, (uint64_t)B}, {128, 512, 2048}, {64, 6, 6, 3});
        const int mB = add_maps(v, v.W3n[n], NB, 2, {64, 576}, {128}, {64, 64});
        if (mA < 0 || mB < 0) return b2g_fail(B2G_ECUDA, "engine v2: cuTensorMapEncodeTiled failed (conv3 dgrad)");
        CgProblem P = kmajor(NB, 64, 9, 3, 108);
        P.nloads = 2;
        P.ld[0] = mk_load(mA, 4, 0); P.ld[0].d_tm[3] = 3; P.ld[0].d_c1[2] = -1; P.ld[0].d_c2[1] = -1;
        P.ld[1] = mk_load(mB, 2, P.b_off); P.ld[1].d_c1[1] = 192; P.ld[1].d_c2[1] = 64;
        P.tiles_m = (B + 2) / 3;
        P.epi = CG_EPI_DGRAD; P.rows_tile = 108; P.lim_rows = B * 36;
        P.o_tm = 108 * 64; P.o0 = 64; P.n_valid = 64; P.out_planes = 2;
        for (int p = 0; p < 2; ++p) P.out_p[p] = v.dZ2[n][p];
        P.mask = v.H2[n][0]; P.m_tm = 108 * 64; P.m0 = 64;
        P.colsum = h->g(h->cnn_t(nets[n], 1, "b")); P.colsum_mask = 63;
        g.host[g.n++] = P;
      }
      {
        const int mA = add_maps(v, v.H2[n], NB, 4, {64, 6, 6, (uint64_t)B}, {128, 768, 4608}, {64, 4, 4, 4});
        const int mB = add_maps(v, v.dZ3[n], NB, 2, {64, (uint64_t)B * 16}, {128}, {64, 64});
        if (mA < 0 || mB < 0) return b2g_fail(B2G_ECUDA, "engine v2: cuTensorMapEncodeTiled failed (conv3 wgrad)");
        CgProblem P = mnmajor(NB, 64, 2, 1, (B + 3) / 4);
        P.nloads = 3;
        for (int a = 0; a < 2; ++a) { P.ld[a] = mk_load(mA, 4, a * P.a_lbo); P.ld[a].d_c2[3] = 4; }
        P.ld[2] = mk_load(mB, 2, P.b_off); P.ld[2].d_c2[1] = 64;
        P.tm_tab = dtab;
        P.tiles_m = 5; P.tiles_n = 1;
        P.splits = std::max(1, std::min(P.chunks, std::max(14, (P.chunks + 15) / 16)));     // <= 16 chunks (64 k-steps) per accumulator chain
        P.lim_rows = 576; P.o_tm = 128 * 64; P.o0 = 64; P.n_valid = 64;
        P.out_f = h->g(h->cnn_t(nets[n], 2, "w")); P.atomic = 1;
        g.host[g.n++] = P;
      }
    }
    if (int rc = push_group(h, v.bwd_groups, g, "conv3_bwd")) return rc;
  }
  // ---- conv2 dgrad: the four output-parity classes of the stride-2 convolution share their A operand (the gradient map
  // shifted by (-jy, -jx), zero-filled outside), so ONE tile computes all four: B = [W(py,px)] stacked along N
  // (4 x 32 input channels = 128 accumulator columns, two boxes of 64 rows), one 32-column group per class, each with
  // its own output offset and row limits (classes with 7 rows / columns mask the 8th).
  {
    CgGroup g;
    for (int n = 0; n < 2; ++n) {
      const int mA = add_maps(v, v.dZ2[n], NB, 4, {64, 6, 6, (uint64_t)B}, {128, 768, 4608}, {64, 8, 8, 2});
      const int mB = add_maps(v, v.W2n[n], NB, 2, {64, 512}, {128}, {64, 64}, {}, false);      // two boxes (py) per plane
      if (mA < 0 || mB < 0) return b2g_fail(B2G_ECUDA, "engine v2: cuTensorMapEncodeTiled failed (conv2 dgrad)");
      CgProblem P = kmajor(NB, 128, 4, 2, 128);
      P.tx_bytes = NB * (128 * 128 + 2 * 64 * 128);
      P.nloads = 3;
      P.ld[0] = mk_load(mA, 4, 0); P.ld[0].d_tm[3] = 2; P.ld[0].d_c1[2] = -1; P.ld[0].d_c2[1] = -1;
      // kernel positions (ky, kx) = (py + 2 jy, px + 2 jx): rows ((2 jy) * 4 + 2 jx) * 32 .. hold (py = 0; px = 0, 1), + 128 rows (py = 1)
      for (int py = 0; py < 2; ++py) {
        P.ld[1 + py] = mk_load(mB, 2, P.b_off + py * 64 * 128);
        P.ld[1 + py].c0[1] = py * 128; P.ld[1 + py].d_c1[1] = 256; P.ld[1 + py].d_c2[1] = 64;
      }
      P.tiles_m = (B + 1) / 2;
      P.epi = CG_EPI_DGRAD; P.rows_tile = 128; P.lim_rows = B * 64;
      P.d0 = 8; P.d1 = 8;
      P.o_tm = 2 * 225 * 64; P.o0 = 2 * 64; P.o1 = 2 * 15 * 64; P.o2 = 225 * 64; P.o_base = n * 32;
      P.m_tm = 2 * 225 * 32; P.m0 = 2 * 32; P.m1 = 2 * 15 * 32; P.m2 = 225 * 32; P.m_base = 0;
      P.grp_tab = 1;
      for (int py = 0; py < 2; ++py)
        for (int px = 0; px < 2; ++px) {
          const int gg = py * 2 + px;
          P.grp_off[gg] = (py * 15 + px) * 64; P.grp_moff[gg] = (py * 15 + px) * 32;
          P.grp_lim0[gg] = (15 - px + 1) / 2; P.grp_lim1[gg] = (15 - py + 1) / 2;
        }
      P.n_valid = 128; P.out_planes = 2;
      for (int p = 0; p < 2; ++p) P.out_p[p] = v.dZ1[p];
      P.mask = v.H1[n][0];
      P.colsum = h->g(h->cnn_t(nets[n], 0, "b")); P.colsum_mask = 31;       // four parity classes x 32 channels
      g.host[g.n++] = P;
    }
    if (int rc = push_group(h, v.bwd_groups, g, "conv2_dgrad")) return rc;
  }
  // ---- conv2 + conv1 wgrad (MN-major, reduction over batch x pixels, split-K with fp32 red.add)
  {
    CgGroup g;
    for (int n = 0; n < 2; ++n) {
      const int mA = add_maps(v, v.H1[n], NB, 4, {64, 14, 15, (uint64_t)B}, {64, 15 * 64, 225 * 64}, {64, 12, 12, 4}, {1, 2, 2, 1});
      const int mB = add_maps(v, v.dZ2[n], NB, 2, {64, (uint64_t)B * 36}, {128}, {64, 144});
      if (mA < 0 || mB < 0) return b2g_fail(B2G_ECUDA, "engine v2: cuTensorMapEncodeTiled failed (conv2 wgrad)");
      CgProblem P = mnmajor(NB, 144, 2, 1, (B + 3) / 4);
      P.nloads = 3;
      for (int a = 0; a < 2; ++a) { P.ld[a] = mk_load(mA, 4, a * P.a_lbo); P.ld[a].c0[1] = 2 * a; P.ld[a].d_tm[2] = 1; P.ld[a].d_c2[3] = 4; }
      P.ld[2] = mk_load(mB, 2, P.b_off); P.ld[2].d_c2[1] = 144;
      P.tiles_m = 4; P.tiles_n = 1;
      P.splits = std::max(1, std::min(P.chunks, std::max(8, (P.chunks + 7) / 8)));           // <= 8 chunks (72 k-steps) per chain
      P.lim_rows = 512; P.o_tm = 128 * 64; P.o0 = 64; P.n_valid = 64;
      P.out_f = h->g(h->cnn_t(nets[n], 1, "w")); P.atomic = 1;
      g.host[g.n++] = P;
    }
    {
      // M = conv1's K rows (window (a, a'), then (b, c, ci)): the M atoms are the shifted S boxes of the forward's views, MN-major.
      // K-chunk (c1, c2) = (sample, band of 4 output rows): the S boxes {.., 16, 4} at block row 16 c1 + 4 c2 + a, and dZ1 viewed
      // as {64, 15 ox, 15 oy, B}, box {64, 16, 4, 1} at (0, 0, 4 c2, c1).  The junk pixels (ox = 15, oy = 15) may be in bounds of
      // S; their dZ1 rows are out of bounds, so they add zeros.
      const int mA = Cp == 1 ? add_maps(v, v.S[0], NB, 3, {32, 15, (uint64_t)B * 16}, {32, 512}, {32, 16, 4}, {}, true, 64)
                             : add_maps(v, v.S[0], NB, 3, {64, 16, (uint64_t)B * 16}, {128, 2048}, {64, 16, 4});
      const int mB = add_maps(v, v.dZ1, NB, 4, {64, 15, 15, (uint64_t)B}, {128, 15 * 128, 225 * 128}, {64, 16, 4, 1});
      if (mA < 0 || mB < 0) return b2g_fail(B2G_ECUDA, "engine v2: cuTensorMapEncodeTiled failed (conv1 wgrad)");
      CgProblem P = mnmajor(NB, 64, 2, 1, 4 * B);
      P.n2 = 4;
      if (Cp == 1) {
        // all four windows (64 rows of M) in one tile: two 32-element atoms (windows (a, 0) | (a, 1)) of 64-byte rows; the second
        // warpgroup repeats the first one's rows (rows 64 .. 127 are not stored)
        P.a_pstride = 64 * 64; P.a_lbo = NB * P.a_pstride;
        P.b_off = 2 * P.a_lbo;
        P.tx_bytes = NB * (2 * 64 * 64 + 64 * 128);
        P.a_kstep = 16 * 64; P.a_kstep2 = 2 * P.a_kstep; P.a_desc = cg_desc_bits(64, true, P.a_lbo); P.a_moff = 0;
        P.nloads = 3;
        for (int a = 0; a < 2; ++a) { P.ld[a] = mk_load(mA, 3, a * P.a_lbo); P.ld[a].c0[2] = a; P.ld[a].d_c1[2] = 16; P.ld[a].d_c2[2] = 4; }
        P.tiles_m = 1;
        P.d0 = 4; P.d1 = 4; P.o0 = 32; P.o1 = 8 * 32;          // row (l, b, c) of window l = 2a + a'
        P.rgrp_rows = 16;
        for (int l = 0; l < 4; ++l) P.rgrp_off[l] = (32 * (l >> 1) + 4 * (l & 1)) * 32;
      } else {
        // tile tm = window row a: the windows (a, 0), (a, 1) as the two 64-wide atoms of the M tile
        for (int l = 0; l < 2; ++l) {
          P.ld[l] = mk_load(mA, 3, l * P.a_lbo); P.ld[l].c0[1] = l; P.ld[l].d_tm[2] = 1; P.ld[l].d_c1[2] = 16; P.ld[l].d_c2[2] = 4;
        }
        P.nloads = 3;
        P.tiles_m = 2;
        P.d0 = 4; P.d1 = 4; P.o0 = 32; P.o1 = Ci * 32; P.o_tm = 32 * Ci * 32;     // row (a', b, c, ci) of window (tm, a')
        P.lim_i0 = Ci;                                         // pad channels
        P.rgrp_rows = 16;
        for (int j = 0; j < 8; ++j) P.rgrp_off[j] = (8 * Ci * (j & 3) + 4 * Ci * (j >> 2)) * 32;
      }
      P.ld[P.nloads - 1] = mk_load(mB, 4, P.b_off); P.ld[P.nloads - 1].d_c1[3] = 1; P.ld[P.nloads - 1].d_c2[2] = 4;
      P.tiles_n = 1;
      P.splits = std::max(1, std::min(P.chunks, std::max(84 / P.tiles_m, (P.chunks + 15) / 16)));
      P.lim_rows = 64 * Cp; P.n_valid = 64;
      P.out_f = h->g(h->cnn_t("model/pi", 0, "w")); P.f_grp = (long long)(h->g(h->cnn_t("model/values_fn", 0, "w")) - h->g(h->cnn_t("model/pi", 0, "w"))); P.atomic = 1;
      g.host[g.n++] = P;
    }
    if (int rc = push_group(h, v.bwd_groups, g, "conv_wgrad")) return rc;
  }
  // ================================================================================ fused launches
  // One persistent launch for the forward chain (conv1 -> conv2 -> conv3 -> cnn_fc1 -> head fc0) and one for the backward chain up
  // to the conv2 dgrad: a launch boundary costs a sizeable share of a layer (launch, first-fetch latency, the last tile's
  // epilogue and the ragged last wave), a counter wait between dependent TILES costs nothing once the pipeline is full.  The stage ring is re-partitioned per problem (the conv2 wgrad needs 108 KB stages, the rest 64 - 72 KB).
  int n_ctr = 0;
  {
    std::vector<const CgGroup*> parts;
    for (auto& g : v.fwd) parts.push_back(&g);                 // conv1 (obs, next), conv2 x3, conv3 x3, fc1 x3, fc0 x3
    std::vector<Wire> w;
    for (int n = 0; n < 3; ++n) {
      w.push_back({1, n, 0, n < 2 ? 0 : 1, 6, 1, 0});          // conv2 tile: 3 samples of H1 = 6 conv1 tiles (two bands per sample)
      w.push_back({2, n, 1, n, 8 * 36, 108, 0});               // conv3 tile: 8 samples of H2 (36 rows each; conv2 tiles are 3 samples)
      w.push_back({3, n, 2, n, 128 * 16, 128, 0});             // fc1 tile: 128 samples of H3 (16 rows each)
      w.push_back({4, n, 3, n, 128, 128, 0});                  // fc0 tile: 128 feature rows (all 8 column tiles of them)
    }
    if (int rc = fuse_groups(h, parts, w, "fwd_fused", v.fwd_fused, n_ctr)) return rc;
  }
  {
    std::vector<const CgGroup*> parts;
    for (auto& g : v.bwd_groups) parts.push_back(&g);          // heads_dgrad, fc1_bwd, conv3_bwd, conv2_dgrad, conv_wgrad
    std::vector<Wire> w;
    for (int n = 0; n < 2; ++n) {
      w.push_back({1, 2 * n, 0, n, 128, 128, 0});              // fc1 dgrad tile: 128 rows of dZ4
      w.push_back({1, 2 * n + 1, 0, n, 64, 128, 1});           // fc1 wgrad chunk: 64 rows of dZ4
      w.push_back({2, 2 * n, 1, 2 * n, 3, 128, 0});            // conv3 dgrad tile: 3 samples of dZ3 (fc1 dgrad rows are samples)
      w.push_back({2, 2 * n + 1, 1, 2 * n, 4, 128, 1});        // conv3 wgrad chunk: 4 samples of dZ3
      w.push_back({3, n, 2, 2 * n, 72, 108, 0});               // conv2 dgrad tile: 2 samples of dZ2 (36 rows each; conv3 dgrad tiles are 3 samples)
      w.push_back({4, n, 2, 2 * n, 144, 108, 1});              // conv2 wgrad chunk: 4 samples of dZ2
    }
    // conv1 wgrad chunk: a quarter sample of dZ1 [B*225][pi | vf]; a conv2 dgrad tile (of EITHER net: both must be done) covers 2 samples
    w.push_back({4, 2, 3, 0, 1, 8, 1});
    w.push_back({4, 2, 3, 1, 1, 8, 1});
    if (int rc = fuse_groups(h, parts, w, "bwd_fused", v.bwd_fused, n_ctr)) return rc;
    // data parallel: the same chain cut after cnn_fc1, where the gradients of [cnn_fc1 .. end] (84 % of the bytes) are final
    // and their all-reduce starts on the side stream underneath the conv backward
    std::vector<const CgGroup*> pa(parts.begin(), parts.begin() + 2), pb(parts.begin() + 2, parts.end());     // pb: conv3_bwd, conv2_dgrad, conv_wgrad
    std::vector<Wire> wa, wb;
    for (int n = 0; n < 2; ++n) {
      wa.push_back({1, 2 * n, 0, n, 128, 128, 0});
      wa.push_back({1, 2 * n + 1, 0, n, 64, 128, 1});
      wb.push_back({1, n, 0, 2 * n, 72, 108, 0});
      wb.push_back({2, n, 0, 2 * n, 144, 108, 1});
    }
    wb.push_back({2, 2, 1, 0, 1, 8, 1});
    wb.push_back({2, 2, 1, 1, 1, 8, 1});
    if (int rc = fuse_groups(h, pa, wa, "bwd_fused_fc", v.bwd_fused, n_ctr)) return rc;
    if (int rc = fuse_groups(h, pb, wb, "bwd_fused_conv", v.bwd_fused, n_ctr)) return rc;
  }
  if (int rc = dev_alloc(h->allocs, h->stream, &v.dep_ctr, (size_t)n_ctr)) return rc;
  v.n_dep_ctr = n_ctr;
  bind_counters(v.fwd_fused, v.dep_ctr);
  bind_counters(v.bwd_fused, v.dep_ctr);
  if (int rc = dev_alloc(h->allocs, h->stream, &v.d_maps, v.maps.size())) return rc;
  CK(cudaMemcpyAsync(v.d_maps, v.maps.data(), v.maps.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}

// ================================================================================================ step pieces
int v2_planes(b2g_sac* h, bool backward, cudaStream_t s) {
  V2State& v = h->v2;
  const int cta0 = backward ? v.plane_ctas_fwd : 0, n = backward ? v.plane_ctas - v.plane_ctas_fwd : v.plane_ctas_fwd;
  planes2_kernel<<<n, 256, 0, s>>>((const Plane2Job*)v.plane_jobs, v.plane_cta_job, cta0);
  return 0;
}

int v2_gather(b2g_sac* h, const GatherArgs& ga, cudaStream_t s) {
  V2State& v = h->v2;
  Gather2Args a{};
  a.g = ga;
  for (int w = 0; w < 2; ++w)
    for (int p = 0; p < 3; ++p) a.s1[w][p] = v.S[w][p];
  for (int n = 0; n < 3; ++n) for (int p = 0; p < 3; ++p) a.fp[n][p] = v.F[n][p];
  a.KF = v.KF;
  const dim3 grid(ga.B, ga.next_obs || ga.next_frame ? 2 : 1);
  switch (h->Cimg) {      // v2 runs 1 .. 4 image channels (sac.cu)
    case 1: gather2_kernel<1><<<grid, 512, 0, s>>>(a); break;
    case 2: gather2_kernel<2><<<grid, 512, 0, s>>>(a); break;
    case 3: gather2_kernel<3><<<grid, 512, 0, s>>>(a); break;
    default: gather2_kernel<4><<<grid, 512, 0, s>>>(a); break;
  }
  return 0;
}

extern long long* g_cg_trace;
static long long* s_trace_buf = nullptr;

int v2_launch(b2g_sac* h, const CgGroup& g, cudaStream_t s) {
  const char* tn = getenv("B2G_CG_TRACE");
  cudaStreamCaptureStatus cs0 = cudaStreamCaptureStatusNone;
  if (tn) cudaStreamIsCapturing(s, &cs0);
  if (tn && cs0 == cudaStreamCaptureStatusNone && std::string(tn) == g.name) {        // bring-up: per-chunk clock64 stamps of CTA 0 -> stderr (serialises the launch)
    if (!s_trace_buf) cudaMalloc(&s_trace_buf, 640 * sizeof(long long));
    cudaMemsetAsync(s_trace_buf, 0, 640 * sizeof(long long), s);
    g_cg_trace = s_trace_buf;
    const char* tc = getenv("B2G_CG_TRACE_CTA");
    cudaError_t e = cg_launch(g, h->v2.d_maps, h->num_sms - h->v2.sm_reserve, s, false, h->v2.dbg | ((tc ? atoi(tc) : 0) << 8));
    g_cg_trace = nullptr;
    if (e != cudaSuccess) return b2g_fail(B2G_ECUDA, cudaGetErrorString(e));
    static int shots = 0;
    if (shots++ == 3) {
      long long t[640];
      cudaStreamSynchronize(s);
      cudaMemcpy(t, s_trace_buf, sizeof(t), cudaMemcpyDeviceToHost);
      const long long t0 = t[0];
      fprintf(stderr, "cg trace %s (cycles; per chunk: prod wait_start wait_done issued | mma wait_start full_seen committed)\n", g.name);
      for (int i = 0; i < 64 && t[i * 8 + 2]; ++i)
        fprintf(stderr, "  chunk %2d (p %lld tm %lld): %7lld %7lld %7lld | %7lld %7lld %7lld\n", i, t[i * 8 + 6] / 100000, t[i * 8 + 6] % 100000 / 10, t[i * 8] - t0,
                t[i * 8 + 1] - t0, t[i * 8 + 2] - t0, t[i * 8 + 3] - t0, t[i * 8 + 4] - t0, t[i * 8 + 5] - t0);
      for (int i = 0; i < 16 && t[512 + i * 4 + 1]; ++i)
        fprintf(stderr, "  tile %d (p %lld tm %lld) mma: start %7lld sums out %7lld (%s)\n", i, t[512 + i * 4 + 3] / 100000, t[512 + i * 4 + 3] % 100000 / 10,
                t[512 + i * 4] - t0, t[512 + i * 4 + 1] - t0, t[512 + i * 4 + 2] ? "handed off" : "in place");
      for (int i = 0; i < 16 && t[576 + i * 4 + 2]; ++i)
        fprintf(stderr, "  handoff %d (p %lld tm %lld) epilogue warpgroup: buffer wait %7lld start %7lld end %7lld\n", i, t[576 + i * 4 + 3] / 100000,
                t[576 + i * 4 + 3] % 100000 / 10, t[576 + i * 4] - t0, t[576 + i * 4 + 1] - t0, t[576 + i * 4 + 2] - t0);
    }
    return 0;
  }
  CK(cg_launch(g, h->v2.d_maps, h->num_sms - h->v2.sm_reserve, s, pdl_enabled(), h->v2.dbg));
  return 0;
}

}  // namespace b2g
