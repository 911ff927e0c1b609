// libb200grasp: convolutional auto-encoder, ENCODER half (forward only) -- SURVEY.md section 8 row a12.
//
// Replaces `SimpleAutoEncoder.encode` (/root/reference/manipulation_main/gripperEnv/encoders.py:59-61, graph
// built at :87-108) as called once per environment step by `EncodedDepthImgSensor.get_state`
// (manipulation_main/gripperEnv/sensor.py:218-222): Conv2D(filters, k, strides, padding='same') + LeakyReLU(alpha)
// per entry of config.yaml's `network`, Flatten, Dense(encoding_dim), LeakyReLU(alpha).
//
// Every layer is one gather-GEMM on the fp32 engine (gg_simt.cu).  TensorFlow 'same' padding is realised by keeping each
// layer's input in a zero-bordered NHWC buffer (enc_tables.cuh): layer l's epilogue writes straight into the interior of
// layer l+1's bordered buffer.  Kernels keep Keras' HWIO layout.
//
// The same launches, over a copy of the tables and weights, make the observation stage of a learner handle (enc_stage.cuh,
// b2g_sac_set_obs_encoder / b2g_bdq_set_obs_encoder): raw rows go in, encoded rows come out in the learner's staging.
//
// Precision B2G_PREC_BF16X3 (b2g_encoder_create2) runs the same four contractions on the wgmma engine (gg_tc.cu, planes mode,
// x3 = 1) instead.  Every layer's input lives as BF16 hi/lo planes: a kernel splits the raw frames into layer 0's planes, each
// hidden layer's epilogue (bias + LeakyReLU) writes its output as hi/lo planes into the interior of the next layer's
// zero-bordered plane buffers, and the dense layer writes fp32 encoded rows.  The cp.async producer copies 16-byte groups of 8
// consecutive reduction elements, so:
//   * layer 0 reads an x-unfolded copy of the image: row (b, y, ox) holds the k * C values one kernel row sees at output
//     column ox, padded with zeros to kp = round8(k * C); its reduction is k * kp long, the padded taps have zero weights;
//   * hidden convs need input channels (the previous conv's filters) % 8 == 0;
//   * the dense layer's input rows are padded to a multiple of 8.
// The weights go to transposed [f, R] planes once per set_weights (planes_launch).  No split-R: every encoding is one tile's
// fixed chain of r-chunks, whatever the batch and the row.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/b200grasp.h"
#include "common.cuh"
#include "enc_stage.cuh"
#include "enc_tables.cuh"
#include "host.cuh"

using namespace b2g;

namespace {
__global__ void enc_pad_copy(const float* __restrict__ src, float* __restrict__ dst, int n, int h, int w, int c, int hp, int wp,
                             int pt, int pl) {
  const long long total = (long long)n * h * w * c;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ch = (int)(i % c);
    long long p = i / c;
    const int x = (int)(p % w); p /= w;
    const int y = (int)(p % h);
    const int b = (int)(p / h);
    dst[(((long long)b * hp + y + pt) * wp + x + pl) * c + ch] = src[i];
  }
}

// The observation stage (enc_stage.cuh).  Raw row r of `raw` ([.][RW] = [P pixels, HWC | T tail floats]) -> layer 0's bordered
// input at sample b, where r = map[b] (or b without a map); the tail goes straight to columns [D, D + T) of encoded row r.
__global__ void enc_stage_in(const float* __restrict__ raw, int RW, const int* __restrict__ map, int n, int w, int c, int hp, int wp,
                             int pt, int pl, float* __restrict__ x, int D, float* __restrict__ dst, int E) {
  const int P = RW - (E - D);
  const long long total = (long long)n * RW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / RW), p = (int)(i - (long long)b * RW);
    const int r = map ? map[b] : b;
    const float v = raw[(long long)r * RW + p];
    if (p < P) {
      const int ch = p % c, q = p / c, xx = q % w, y = q / w;
      x[(((long long)b * hp + y + pt) * wp + xx + pl) * c + ch] = v;
    } else {
      dst[(long long)r * E + D + (p - P)] = v;
    }
  }
}

// encoding of sample b (z row b) -> columns [0, D) of encoded row map[b] (or b)
__global__ void enc_stage_out(const float* __restrict__ z, int zs, const int* __restrict__ map, int n, int D, float* __restrict__ dst,
                              int E) {
  const long long total = (long long)n * D;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / D), e = (int)(i - (long long)b * D);
    dst[(long long)(map ? map[b] : b) * E + e] = z[(long long)b * zs + e];
  }
}

// Raw rows -> layer 0's x-unfolded BF16 hi/lo planes [n][hp][ow][kp] (bf16x3).  Element (b, y, ox, j) is channel j % c of
// pixel (y - pt, ox * s + j / c - pl) of raw row r = map[b] (or b) when j < k * c and the pixel lies in the image, else 0.
// One thread per 8 elements (16 bytes of each plane).  Threads past the planes copy the row's tail floats [P, RW) to columns
// [D, D + T) of encoded row r, as enc_stage_in does (dst == nullptr: no tail).
__global__ void enc_split_in(const float* __restrict__ raw, int RW, const int* __restrict__ map, int n, int h, int w, int c, int k,
                             int s, int hp, int ow, int kp, int pt, int pl, uint16_t* __restrict__ hi, uint16_t* __restrict__ lo, int D,
                             float* __restrict__ dst, int E) {
  const int T = E - D, P = RW - T, kc = k * c, g8 = kp / 8;
  const long long groups = (long long)n * hp * ow * g8, total = groups + (dst ? (long long)n * T : 0);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    if (i >= groups) {
      const long long t = i - groups;
      const int b = (int)(t / T), p = (int)(t - (long long)b * T);
      const int r = map ? map[b] : b;
      dst[(long long)r * E + D + p] = raw[(long long)r * RW + P + p];
      continue;
    }
    long long q = i;
    const int j0 = (int)(q % g8) * 8; q /= g8;
    const int ox = (int)(q % ow); q /= ow;
    const int y = (int)(q % hp);
    const int b = (int)(q / hp);
    const int r = map ? map[b] : b;
    const float* row = raw + (long long)r * RW;
    const int yy = y - pt;
    uint32_t hw[4], lw[4];
#pragma unroll
    for (int e = 0; e < 8; e += 2) {
      float v[2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int j = j0 + e + u, xx = ox * s + j / c - pl;
        v[u] = (j < kc && yy >= 0 && yy < h && xx >= 0 && xx < w) ? row[(yy * w + xx) * c + j % c] : 0.f;
      }
      const __nv_bfloat16 h0 = __float2bfloat16_rn(v[0]), h1 = __float2bfloat16_rn(v[1]);
      const __nv_bfloat16 l0 = __float2bfloat16_rn(v[0] - __bfloat162float(h0)), l1 = __float2bfloat16_rn(v[1] - __bfloat162float(h1));
      hw[e / 2] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
      lw[e / 2] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
    }
    *reinterpret_cast<uint4*>(hi + i * 8) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
    *reinterpret_cast<uint4*>(lo + i * 8) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
  }
}

// map[j] = index of the j-th finished env (done[i] != 0), i < n
__global__ void enc_done_map(const float* __restrict__ done, int n, int* __restrict__ map) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  int j = 0;
  for (int i = 0; i < n; ++i)
    if (done[i] != 0.f) map[j++] = i;
}
}  // namespace

namespace b2g {
// bf16x3: one layer's BF16 planes and its reduction on the wgmma engine
struct EncPlanes {
  int Rt = 0;                  // reduction length: layer 0 k * kp, hidden convs k * k * in_c, dense R
  int ws = 0;                  // row stride of the weight planes: round8(Rt), so every row starts 16-byte aligned
  int kp = 0;                  // layer 0: taps per unfolded kernel row (round8(k * C))
  int rs = 0;                  // dense: row stride of its input planes (round8(R))
  size_t in_per = 0;           // input plane elements per sample
  uint16_t* in_hi = nullptr; uint16_t* in_lo = nullptr;   // input planes [N][in_per]
  uint16_t* w_hi = nullptr; uint16_t* w_lo = nullptr;     // weight planes [fs][ws]
  float* wq = nullptr;         // [ws][fs] fp32 weights in the engine's r order, zero rows from Rt on (the planes' source)
  PlaneJob* job = nullptr;     // device copy of the planes_launch job
};
}  // namespace b2g

struct b2g_encoder {
  b2g_encoder_cfg cfg{};
  int precision = B2G_PREC_FP32_SIMT;
  int num_sms = 0;
  cudaStream_t stream = nullptr;
  std::vector<void*> allocs;
  std::vector<EncLayer> layers;          // convs then the dense layer
  std::vector<EncPlanes> planes;         // bf16x3: per layer
  float* stage_in = nullptr;             // [N, H, W, C] as received
  float* z = nullptr;                    // [N, zs]
  int zs = 0;
  std::vector<GemmGroup> groups;         // one launch per layer (each consumes the previous one's output)
  int built_n = -1;
  float* pin_in = nullptr;
  float* pin_out = nullptr;
};

namespace {
constexpr int ENC_TC_FLAGS = GG_PLANES | GG_EPI_BIAS_LRELU;   // selects gg_tc's encoder instantiation

int round_up(int x, int m) { return (x + m - 1) / m * m; }

// The bf16x3 plane geometry of `layers` (sizes only; no memory).  0, or B2G_EINVAL with the reason set.
int tc_geometry(const std::vector<EncLayer>& layers, std::vector<EncPlanes>& planes) {
  const int L = (int)layers.size();
  planes.assign(L, EncPlanes{});
  for (int l = 0; l < L; ++l) {
    const EncLayer& y = layers[l];
    EncPlanes& p = planes[l];
    if (y.k == 0) {
      p.Rt = y.R(); p.rs = round_up(p.Rt, 8); p.in_per = p.rs;
    } else if (l == 0) {
      p.kp = round_up(y.k * y.in_c, 8); p.Rt = y.k * p.kp; p.in_per = (size_t)y.hp * y.out_w * p.kp;
    } else {
      if (y.in_c % 8)
        return b2g_fail(B2G_EINVAL, "bf16x3: conv layer " + std::to_string(l - 1) + " has " + std::to_string(y.in_c) +
                                        " filters; the next conv reads them as BF16 plane rows of 8-channel (16-byte) groups, so "
                                        "every conv but the last needs filters % 8 == 0");
      p.Rt = y.R(); p.in_per = (size_t)y.hp * y.wp * y.in_c;
    }
    p.ws = round_up(p.Rt, 8);
  }
  return 0;
}

// Largest element offset any bf16x3 table of N samples addresses (checked against 2^31 - 1 at create).
size_t tc_biggest(const std::vector<EncLayer>& layers, const std::vector<EncPlanes>& planes, size_t N) {
  size_t b = 0;
  for (size_t l = 0; l < layers.size(); ++l) b = std::max(b, N * planes[l].in_per);
  return b;
}

// Device memory of the bf16x3 planes for N samples (input planes zeroed: the borders stay zero), and the weight planes.
int tc_alloc(const std::vector<EncLayer>& layers, std::vector<EncPlanes>& planes, size_t N, std::vector<void*>& allocs, cudaStream_t s) {
  for (size_t l = 0; l < layers.size(); ++l) {
    EncPlanes& p = planes[l];
    if (int rc = dev_alloc(allocs, s, &p.in_hi, N * p.in_per)) return rc;
    if (int rc = dev_alloc(allocs, s, &p.in_lo, N * p.in_per)) return rc;
    if (int rc = dev_alloc(allocs, s, &p.w_hi, (size_t)layers[l].fs * p.ws)) return rc;
    if (int rc = dev_alloc(allocs, s, &p.w_lo, (size_t)layers[l].fs * p.ws)) return rc;
  }
  return 0;
}

// Tile grid of a one-descriptor wgmma launch (the descriptor travels by value: nothing to upload).
void tc_tiles(GemmGroup& g) {
  GemmDesc& d = g.host[0];
  d.tiles_m = (d.M + GG_TC_BM - 1) / GG_TC_BM;
  d.tiles_n = (d.N + GG_TC_BN - 1) / GG_TC_BN;
  d.tile_start = 0;
  d.tile_count = d.tiles_m * d.tiles_n;
  g.total_tiles = d.tile_count;
}

// The bf16x3 launches of an encoder's layers over N samples: layer l reads planes[l].in_*, a conv writes the interior of the next
// layer's input planes (C_hi / C_lo only), the dense layer fp32 rows of `out_dense` at stride `out_stride`.
int build_tc_tables(const std::vector<EncLayer>& layers, const std::vector<EncPlanes>& planes, int N, float alpha, float* out_dense,
                    int out_stride, std::vector<GemmGroup>& groups, std::vector<void*>& allocs, cudaStream_t s) {
  const int L = (int)layers.size();
  groups.assign(L, GemmGroup{});
  for (int l = 0; l < L; ++l) {
    const EncLayer& y = layers[l];
    const EncPlanes& p = planes[l];
    const bool dense = y.k == 0;
    const int M = N * y.out_h * y.out_w, Rt = p.Rt, Rpad = round_up(Rt, GG_TC_BK);
    std::vector<int> aM(M), cM(M), aR(Rpad, 0), bR(Rpad, 0), bN(y.f), cN(y.f);
    for (int b = 0; b < N; ++b)
      for (int oy = 0; oy < y.out_h; ++oy)
        for (int ox = 0; ox < y.out_w; ++ox) {
          const int m = (b * y.out_h + oy) * y.out_w + ox;
          if (dense) aM[m] = b * p.rs;
          else if (l == 0) aM[m] = ((b * y.hp + oy * y.s) * y.out_w + ox) * p.kp;
          else aM[m] = ((b * y.hp + oy * y.s) * y.wp + ox * y.s) * y.in_c;
          if (dense) cM[m] = b * out_stride;
          else if (layers[l + 1].k == 0) cM[m] = b * planes[l + 1].rs + (oy * y.out_w + ox) * y.f;
          else {
            const EncLayer& nx = layers[l + 1];
            cM[m] = ((b * nx.hp + oy + nx.pad_t) * nx.wp + ox + nx.pad_l) * y.f;
          }
        }
    for (int r = 0; r < Rt; ++r) {
      if (dense) aR[r] = r;
      else if (l == 0) aR[r] = (r / p.kp) * y.out_w * p.kp + r % p.kp;
      else {
        const int c = r % y.in_c, kx = (r / y.in_c) % y.k, ky = r / (y.in_c * y.k);
        aR[r] = (ky * y.wp + kx) * y.in_c + c;
      }
      bR[r] = r;
    }
    for (int n = 0; n < y.f; ++n) { bN[n] = n * p.ws; cN[n] = n; }
    GemmDesc d = gemm_desc(nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, dense ? out_dense : nullptr, nullptr, nullptr, M, y.f,
                           Rt, ENC_TC_FLAGS);
    d.bias = y.b; d.alpha = alpha;
    d.A_hi = p.in_hi; d.A_lo = p.in_lo; d.B_hi = p.w_hi; d.B_lo = p.w_lo;
    if (!dense) { d.C_hi = planes[l + 1].in_hi; d.C_lo = planes[l + 1].in_lo; }
    std::map<const int*, std::vector<int>> host;
    if (int rc = upload_table(allocs, s, aM, &d.aM)) return rc;
    if (int rc = upload_table(allocs, s, aR, &d.aR)) return rc;
    if (int rc = upload_table(allocs, s, bR, &d.bR_p)) return rc;
    if (int rc = upload_table(allocs, s, bN, &d.bN_p)) return rc;
    if (int rc = upload_table(allocs, s, cM, &d.cM, &host)) return rc;
    if (int rc = upload_table(allocs, s, cN, &d.cN, &host)) return rc;
    ColIds ids;
    gg_tc_columns(d, host, ids);
    GemmGroup& g = groups[l];
    g.name = dense ? "enc_dense_tc" : "enc_conv" + std::to_string(l) + "_tc";
    g.host = {d};
    g.tc = true;
    tc_tiles(g);
  }
  return 0;
}

// Raw rows (or images, tail 0) -> layer 0's planes, then every layer on the wgmma engine.
int tc_forward(const std::vector<EncLayer>& layers, const std::vector<EncPlanes>& planes, std::vector<GemmGroup>& groups,
               const b2g_encoder_cfg& cfg, const float* raw, int RW, const int* map, int n, float* dst, int E, int num_sms,
               cudaStream_t s) {
  const EncLayer& y0 = layers[0];
  const EncPlanes& p0 = planes[0];
  const long long work = (long long)n * p0.in_per / 8 + (dst ? (long long)n * (E - cfg.encoding_dim) : 0);
  const int blocks = (int)std::min<long long>((work + 255) / 256, 132 * 8);
  enc_split_in<<<blocks, 256, 0, s>>>(raw, RW, map, n, cfg.height, cfg.width, cfg.channels, y0.k, y0.s, y0.hp, y0.out_w, p0.kp,
                                      y0.pad_t, y0.pad_l, p0.in_hi, p0.in_lo, cfg.encoding_dim, dst, E);
  CK(cudaGetLastError());
  for (auto& g : groups) CK(gg_tc_launch(g.host.data(), 1, g.total_tiles, ENC_TC_FLAGS, 1, num_sms, s));
  return 0;
}

// The forward launches of an encoder's layers over N samples (tables for the whole capacity; a call with n < N uses the leading
// n * out_h * out_w rows): a conv layer writes the interior of the next layer's bordered input, the dense layer rows of `out`
// at row stride `out_stride`.  Shared by the encoder handle (out = z) and the observation stage of a learner handle.
int build_tables(std::vector<EncLayer>& layers, int N, float alpha, float* out_dense, int out_stride, std::vector<GemmGroup>& groups,
                 std::vector<void*>& allocs, cudaStream_t s) {
  const int L = (int)layers.size();
  groups.resize(L);
  for (int l = 0; l < L; ++l) {
    EncLayer& y = layers[l];
    const bool dense = y.k == 0;
    // where this layer's output lands: interior of the next layer's bordered input, or the dense output rows
    float* out;
    int o_hp, o_wp, o_pt, o_pl, o_c;
    if (dense) { out = out_dense; o_hp = o_wp = 1; o_pt = o_pl = 0; o_c = out_stride; }
    else {
      const EncLayer& nx = layers[l + 1];
      out = nx.in; o_hp = nx.hp; o_wp = nx.wp; o_pt = nx.pad_t; o_pl = nx.pad_l; o_c = y.f;
    }
    const int M = N * y.out_h * y.out_w, R = y.R();
    std::vector<int> aM, cM, aR, bR, bN, cN;
    enc_fwd_tables(y, N, o_hp, o_wp, o_pt, o_pl, o_c, aM, cM, aR, bR, bN, cN);
    GemmDesc d = gemm_desc(y.in, nullptr, nullptr, y.w, nullptr, nullptr, out, nullptr, nullptr, M, y.f, R, enc_fwd_flags(y));
    d.bias = y.b; d.alpha = alpha;
    if (int rc = upload_table(allocs, s, aM, &d.aM)) return rc;
    if (int rc = upload_table(allocs, s, aR, &d.aR)) return rc;
    if (int rc = upload_table(allocs, s, bR, &d.bR)) return rc;
    if (int rc = upload_table(allocs, s, bN, &d.bN)) return rc;
    if (int rc = upload_table(allocs, s, cM, &d.cM)) return rc;
    if (int rc = upload_table(allocs, s, cN, &d.cN)) return rc;
    GemmGroup& g = groups[l];
    g.name = dense ? "enc_dense" : "enc_conv" + std::to_string(l);
    g.host = {d};
    if (int rc = finalize_tiles(g, allocs, s)) return rc;
  }
  return 0;
}

// The groups' descriptors for the leading n samples; built_n is the batch they currently describe.
int set_batch(const std::vector<EncLayer>& layers, std::vector<GemmGroup>& groups, int& built_n, int n, std::vector<void*>& allocs,
              cudaStream_t s) {
  if (built_n == n) return 0;
  for (size_t l = 0; l < layers.size(); ++l) {
    const EncLayer& y = layers[l];
    groups[l].host[0].M = n * y.out_h * y.out_w;
    if (groups[l].tc) tc_tiles(groups[l]);
    else if (int rc = finalize_tiles(groups[l], allocs, s)) return rc;
  }
  built_n = n;
  return 0;
}
}  // namespace

extern "C" {

int b2g_encoder_create(const b2g_encoder_cfg* cfg, b2g_encoder** out) { return b2g_encoder_create2(cfg, B2G_PREC_FP32_SIMT, out); }

int b2g_encoder_create2(const b2g_encoder_cfg* cfg, int32_t precision, b2g_encoder** out) {
  if (!cfg || !out) return b2g_fail(B2G_EINVAL, "null argument");
  if (precision == B2G_PREC_BF16)
    return b2g_fail(B2G_EINVAL, "encoder precision B2G_PREC_BF16: single-pass BF16 encodings are not offered as policy inputs; use "
                                "B2G_PREC_FP32_SIMT or B2G_PREC_BF16X3");
  if (precision != B2G_PREC_FP32_SIMT && precision != B2G_PREC_BF16X3)
    return b2g_fail(B2G_EINVAL, "encoder precision " + std::to_string(precision) + ": expected B2G_PREC_FP32_SIMT (0) or B2G_PREC_BF16X3 (1)");
  if (cfg->n_layers < 1 || cfg->n_layers > B2G_ENC_MAX_LAYERS) return b2g_fail(B2G_EINVAL, "n_layers out of range");
  if (cfg->height < 1 || cfg->width < 1 || cfg->channels < 1 || cfg->encoding_dim < 1 || cfg->max_batch < 1)
    return b2g_fail(B2G_EINVAL, "non-positive dimension");
  std::vector<EncLayer> layers;
  if (int rc = enc_geometry(*cfg, layers)) return rc;
  const size_t N = cfg->max_batch;
  // every offset table is int: each layer's bordered input (the dense layer's is the flattened last conv output) and z
  size_t biggest = N * (size_t)layers.back().fs;
  for (const auto& y : layers) biggest = std::max(biggest, N * y.hp * y.wp * y.in_c);
  if (biggest > (size_t)((1u << 31) - 1)) return b2g_fail(B2G_EINVAL, "max_batch too large for 32-bit offset tables");
  std::vector<EncPlanes> planes;
  if (precision == B2G_PREC_BF16X3) {
    if (int rc = tc_geometry(layers, planes)) return rc;
    if (tc_biggest(layers, planes, N) > (size_t)((1u << 31) - 1))
      return b2g_fail(B2G_EINVAL, "bf16x3: max_batch too large for 32-bit offset tables of layer 0's unfolded planes");
  }
  int num_sms = 0;
  if (int rc = check_device(cfg->device, &num_sms)) return rc;
  b2g_encoder* h = new b2g_encoder();
  h->cfg = *cfg;
  h->precision = precision;
  h->num_sms = num_sms;
  h->layers = layers;
  h->planes = planes;
  auto bail = [&](int rc) { b2g_encoder_destroy(h); return rc; };
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "stream create"));
  const EncLayer& dn = h->layers.back();
  int rc;
  for (auto& y : h->layers) {
    if ((rc = dev_alloc(h->allocs, h->stream, &y.in, N * y.hp * y.wp * y.in_c))) return bail(rc);
    if ((rc = dev_alloc(h->allocs, h->stream, &y.w, (size_t)y.R() * y.fs))) return bail(rc);
    if ((rc = dev_alloc(h->allocs, h->stream, &y.b, (size_t)y.fs))) return bail(rc);
  }
  h->zs = dn.fs;
  if ((rc = dev_alloc(h->allocs, h->stream, &h->stage_in, N * cfg->height * cfg->width * cfg->channels))) return bail(rc);
  if ((rc = dev_alloc(h->allocs, h->stream, &h->z, N * h->zs))) return bail(rc);
  if (cudaMallocHost(&h->pin_in, N * cfg->height * cfg->width * cfg->channels * sizeof(float)) != cudaSuccess ||
      cudaMallocHost(&h->pin_out, N * cfg->encoding_dim * sizeof(float)) != cudaSuccess)
    return bail(b2g_fail(B2G_ECUDA, "pinned staging allocation failed"));
  if (precision == B2G_PREC_BF16X3) {
    if ((rc = tc_alloc(h->layers, h->planes, N, h->allocs, h->stream))) return bail(rc);
    for (size_t l = 0; l < h->layers.size(); ++l) {
      EncPlanes& p = h->planes[l];
      if ((rc = dev_alloc(h->allocs, h->stream, &p.wq, (size_t)p.ws * h->layers[l].fs))) return bail(rc);
      if ((rc = dev_alloc(h->allocs, h->stream, &p.job, 1))) return bail(rc);
    }
    if ((rc = build_tc_tables(h->layers, h->planes, (int)N, h->cfg.alpha, h->z, h->zs, h->groups, h->allocs, h->stream))) return bail(rc);
  } else if ((rc = build_tables(h->layers, (int)N, h->cfg.alpha, h->z, h->zs, h->groups, h->allocs, h->stream))) {
    return bail(rc);
  }
  h->built_n = (int)N;
  if (cudaStreamSynchronize(h->stream) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "encoder create sync"));
  *out = h;
  return 0;
}

int b2g_encoder_destroy(b2g_encoder* h) {
  if (!h) return 0;
  cudaSetDevice(h->cfg.device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (void* p : h->allocs) cudaFree(p);
  if (h->pin_in) cudaFreeHost(h->pin_in);
  if (h->pin_out) cudaFreeHost(h->pin_out);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

int b2g_encoder_n_layers(const b2g_encoder* h) { return h ? (int)h->layers.size() : -1; }

int b2g_encoder_layer_shape(const b2g_encoder* h, int layer, int64_t* kernel_numel, int64_t* bias_numel) {
  if (!h || layer < 0 || layer >= (int)h->layers.size()) return b2g_fail(B2G_EINVAL, "layer out of range");
  const EncLayer& y = h->layers[layer];
  if (kernel_numel) *kernel_numel = (int64_t)y.R() * y.f;
  if (bias_numel) *bias_numel = y.f;
  return 0;
}

int b2g_encoder_set_weights(b2g_encoder* h, int layer, const float* kernel, size_t kernel_numel, const float* bias, size_t bias_numel) {
  if (!h || !kernel || !bias) return b2g_fail(B2G_EINVAL, "null argument");
  if (layer < 0 || layer >= (int)h->layers.size()) return b2g_fail(B2G_EINVAL, "layer out of range");
  EncLayer& y = h->layers[layer];
  if (kernel_numel != (size_t)y.R() * y.f || bias_numel != (size_t)y.f)
    return b2g_fail(B2G_EINVAL, "layer " + std::to_string(layer) + ": expected kernel numel " + std::to_string((size_t)y.R() * y.f) +
                                 ", bias numel " + std::to_string(y.f));
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemcpy2DAsync(y.w, y.fs * sizeof(float), kernel, y.f * sizeof(float), y.f * sizeof(float), y.R(), cudaMemcpyHostToDevice,
                        h->stream));
  CK(cudaMemcpyAsync(y.b, bias, y.f * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  if (h->precision == B2G_PREC_BF16X3) {
    // [ws][fs] in the engine's r order (layer 0: row ky * kp + j holds tap (ky, j / C, j % C), zero for j >= k * C; zero rows
    // from Rt on), then the transposed hi/lo planes [fs][ws]
    EncPlanes& p = h->planes[layer];
    std::vector<float> wq((size_t)p.ws * y.fs, 0.f);
    for (int r = 0; r < p.Rt; ++r) {
      int src = r;
      if (layer == 0) {
        const int ky = r / p.kp, j = r % p.kp;
        src = j < y.k * y.in_c ? (ky * y.k + j / y.in_c) * y.in_c + j % y.in_c : -1;
      }
      if (src >= 0) memcpy(&wq[(size_t)r * y.fs], kernel + (size_t)src * y.f, y.f * sizeof(float));
    }
    PlaneJob job{};
    job.src = p.wq; job.hiT = p.w_hi; job.loT = p.w_lo; job.R = p.ws; job.N = y.fs; job.tile_start = 0;
    CK(cudaMemcpyAsync(p.wq, wq.data(), wq.size() * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(p.job, &job, sizeof(job), cudaMemcpyHostToDevice, h->stream));
    planes_launch(p.job, 1, ((p.ws + 31) / 32) * ((y.fs + 31) / 32), h->stream);
    CK(cudaGetLastError());
  }
  CK(cudaStreamSynchronize(h->stream));
  y.loaded = true;
  return 0;
}

int b2g_encoder_encode(b2g_encoder* h, const float* imgs, int n, float* out) {
  if (!h || !imgs || !out) return b2g_fail(B2G_EINVAL, "null argument");
  if (n < 1 || n > h->cfg.max_batch) return b2g_fail(B2G_EINVAL, "batch " + std::to_string(n) + " outside [1, max_batch]");
  for (size_t l = 0; l < h->layers.size(); ++l)
    if (!h->layers[l].loaded) return b2g_fail(B2G_ESTATE, "encoder layer " + std::to_string(l) + " has no weights (load_weights first)");
  CK(cudaSetDevice(h->cfg.device));
  if (int rc = set_batch(h->layers, h->groups, h->built_n, n, h->allocs, h->stream)) return rc;
  const EncLayer& y0 = h->layers[0];
  const int hwc = h->cfg.height * h->cfg.width * h->cfg.channels;
  const size_t in_numel = (size_t)n * hwc;
  memcpy(h->pin_in, imgs, in_numel * sizeof(float));
  CK(cudaMemcpyAsync(h->stage_in, h->pin_in, in_numel * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  if (h->precision == B2G_PREC_BF16X3) {
    if (int rc = tc_forward(h->layers, h->planes, h->groups, h->cfg, h->stage_in, hwc, nullptr, n, nullptr, h->cfg.encoding_dim,
                            h->num_sms, h->stream))
      return rc;
  } else {
    const int blocks = (int)std::min<size_t>((in_numel + 255) / 256, 132 * 8);
    enc_pad_copy<<<blocks, 256, 0, h->stream>>>(h->stage_in, y0.in, n, h->cfg.height, h->cfg.width, h->cfg.channels, y0.hp, y0.wp,
                                                y0.pad_t, y0.pad_l);
    for (auto& g : h->groups) gg_simt_launch(g.dev, 1, g.total_tiles, h->stream);
    CK(cudaGetLastError());
  }
  CK(cudaMemcpy2DAsync(h->pin_out, h->cfg.encoding_dim * sizeof(float), h->z, h->zs * sizeof(float),
                        h->cfg.encoding_dim * sizeof(float), n, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  memcpy(out, h->pin_out, (size_t)n * h->cfg.encoding_dim * sizeof(float));
  return 0;
}

int b2g_debug_encoder_layers(b2g_encoder* h, const float* imgs, int n, float* out, int64_t out_numel) {
  if (!h || !imgs || !out) return b2g_fail(B2G_EINVAL, "null argument");
  const int L = (int)h->layers.size();
  int64_t want = 0;
  for (int l = 0; l < L; ++l) want += (int64_t)n * h->layers[l].out_h * h->layers[l].out_w * h->layers[l].f;
  if (out_numel != want) return b2g_fail(B2G_EINVAL, "out_numel " + std::to_string(out_numel) + " != " + std::to_string(want));
  float* z = out + (want - (int64_t)n * h->cfg.encoding_dim);
  if (int rc = b2g_encoder_encode(h, imgs, n, z)) return rc;
  float* o = out;
  for (int l = 0; l + 1 < L; ++l) {      // conv l's output: the interior of layer l + 1's input, [n][out_h][out_w][f]
    const EncLayer& y = h->layers[l];
    const EncLayer& nx = h->layers[l + 1];
    const bool tc = h->precision == B2G_PREC_BF16X3;
    const size_t per = tc ? h->planes[l + 1].in_per : (size_t)nx.hp * nx.wp * nx.in_c;
    std::vector<float> f32;
    std::vector<uint16_t> hi, lo;
    if (tc) {
      hi.resize((size_t)n * per); lo.resize((size_t)n * per);
      CK(cudaMemcpy(hi.data(), h->planes[l + 1].in_hi, hi.size() * 2, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(lo.data(), h->planes[l + 1].in_lo, lo.size() * 2, cudaMemcpyDeviceToHost));
    } else {
      f32.resize((size_t)n * per);
      CK(cudaMemcpy(f32.data(), nx.in, f32.size() * 4, cudaMemcpyDeviceToHost));
    }
    auto bf = [](uint16_t u) { uint32_t v = (uint32_t)u << 16; float f; memcpy(&f, &v, 4); return f; };
    for (int b = 0; b < n; ++b)
      for (int oy = 0; oy < y.out_h; ++oy)
        for (int ox = 0; ox < y.out_w; ++ox)
          for (int c = 0; c < y.f; ++c) {
            size_t e;
            if (nx.k == 0) e = (size_t)b * (tc ? h->planes[l + 1].rs : nx.R()) + (size_t)(oy * y.out_w + ox) * y.f + c;
            else e = (size_t)b * per + ((size_t)(oy + nx.pad_t) * nx.wp + ox + nx.pad_l) * y.f + c;
            *o++ = tc ? bf(hi[e]) + bf(lo[e]) : f32[e];
          }
  }
  return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ observation stage of a learner
namespace b2g {

struct EncStage {
  b2g_encoder_cfg cfg{};           // the encoder's, with max_batch = the learner's staging rows
  int tail = 0, RW = 0, E = 0;     // raw row floats (H*W*C + tail), encoded row floats (encoding_dim + tail)
  std::vector<void*> allocs;
  std::vector<EncLayer> layers;
  int precision = B2G_PREC_FP32_SIMT;   // the encoder's
  int num_sms = 0;
  std::vector<EncPlanes> planes;   // bf16x3: per layer
  float* z = nullptr;              // [rows][zs]
  int zs = 0;
  float* raw[2]{};                 // [rows][RW]: 0 = every env's frame, 1 = reset frames of finished envs (row = env)
  int* map = nullptr;              // [rows]: env of the j-th finished env
  // the same tables, two descriptor sets: the batch of every env and that of the finished envs change independently, so
  // neither re-finalises when only the other changes
  std::vector<GemmGroup> groups[2];
  int built_n[2] = {-1, -1};
};

int enc_stage_check(const b2g_encoder* enc, int device, int tail, int obs_dim) {
  if (tail < 0) return b2g_fail(B2G_EINVAL, "set_obs_encoder: tail must be >= 0");
  if (enc->cfg.encoding_dim + tail != obs_dim)
    return b2g_fail(B2G_EINVAL, "set_obs_encoder: encoding_dim " + std::to_string(enc->cfg.encoding_dim) + " + tail " +
                                    std::to_string(tail) + " != the learner's obs_dim " + std::to_string(obs_dim));
  if (enc->cfg.device != device) return b2g_fail(B2G_EINVAL, "set_obs_encoder: the encoder lives on another device");
  for (size_t l = 0; l < enc->layers.size(); ++l)
    if (!enc->layers[l].loaded)
      return b2g_fail(B2G_ESTATE, "set_obs_encoder: encoder layer " + std::to_string(l) + " has no weights (load_weights first)");
  return 0;
}

int enc_stage_create(const b2g_encoder* enc, int rows, int tail, cudaStream_t s, EncStage** out) {
  const size_t N = rows;
  size_t biggest = N * (size_t)enc->layers.back().fs;
  for (const auto& y : enc->layers) biggest = std::max(biggest, N * y.hp * y.wp * y.in_c);
  if (biggest > (size_t)((1u << 31) - 1)) return b2g_fail(B2G_EINVAL, "set_obs_encoder: staging rows too many for 32-bit offset tables");
  EncStage* st = new EncStage();
  st->cfg = enc->cfg;
  st->cfg.max_batch = rows;
  st->tail = tail;
  st->RW = enc->cfg.height * enc->cfg.width * enc->cfg.channels + tail;
  st->E = enc->cfg.encoding_dim + tail;
  st->layers = enc->layers;
  st->precision = enc->precision;
  st->planes = enc->planes;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&st->num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
    delete st;
    return b2g_fail(B2G_ECUDA, "set_obs_encoder: device attributes");
  }
  if (st->precision == B2G_PREC_BF16X3 && tc_biggest(st->layers, st->planes, N) > (size_t)((1u << 31) - 1)) {
    delete st;
    return b2g_fail(B2G_EINVAL, "set_obs_encoder: staging rows too many for 32-bit offset tables of layer 0's unfolded planes");
  }
  auto bail = [&](int rc) { cudaStreamSynchronize(s); enc_stage_destroy(st); return rc; };
  int rc;
  for (size_t l = 0; l < st->layers.size(); ++l) {      // weights device to device: frozen, the encoder handle may go away
    EncLayer& y = st->layers[l];
    const EncLayer& src = enc->layers[l];
    if ((rc = dev_alloc(st->allocs, s, &y.in, N * y.hp * y.wp * y.in_c))) return bail(rc);
    if ((rc = dev_alloc(st->allocs, s, &y.w, (size_t)y.R() * y.fs))) return bail(rc);
    if ((rc = dev_alloc(st->allocs, s, &y.b, (size_t)y.fs))) return bail(rc);
    if (cudaMemcpyAsync(y.w, src.w, (size_t)y.R() * y.fs * sizeof(float), cudaMemcpyDeviceToDevice, s) != cudaSuccess ||
        cudaMemcpyAsync(y.b, src.b, (size_t)y.fs * sizeof(float), cudaMemcpyDeviceToDevice, s) != cudaSuccess)
      return bail(b2g_fail(B2G_ECUDA, "set_obs_encoder: weight copy"));
  }
  st->zs = st->layers.back().fs;
  if ((rc = dev_alloc(st->allocs, s, &st->z, N * st->zs))) return bail(rc);
  for (int k = 0; k < 2; ++k)
    if ((rc = dev_alloc(st->allocs, s, &st->raw[k], N * st->RW))) return bail(rc);
  if ((rc = dev_alloc(st->allocs, s, &st->map, N))) return bail(rc);
  if (st->precision == B2G_PREC_BF16X3) {      // the encoder's weight planes, device to device; input planes of its own
    if ((rc = tc_alloc(st->layers, st->planes, N, st->allocs, s))) return bail(rc);
    for (size_t l = 0; l < st->layers.size(); ++l) {
      const size_t wn = (size_t)st->layers[l].fs * st->planes[l].ws;
      st->planes[l].wq = nullptr; st->planes[l].job = nullptr;
      if (cudaMemcpyAsync(st->planes[l].w_hi, enc->planes[l].w_hi, wn * 2, cudaMemcpyDeviceToDevice, s) != cudaSuccess ||
          cudaMemcpyAsync(st->planes[l].w_lo, enc->planes[l].w_lo, wn * 2, cudaMemcpyDeviceToDevice, s) != cudaSuccess)
        return bail(b2g_fail(B2G_ECUDA, "set_obs_encoder: weight plane copy"));
    }
    if ((rc = build_tc_tables(st->layers, st->planes, rows, st->cfg.alpha, st->z, st->zs, st->groups[0], st->allocs, s))) return bail(rc);
  } else if ((rc = build_tables(st->layers, rows, st->cfg.alpha, st->z, st->zs, st->groups[0], st->allocs, s))) {
    return bail(rc);
  }
  st->built_n[0] = rows;
  st->groups[1] = st->groups[0];
  for (auto& g : st->groups[1]) g.dev = nullptr;       // its own descriptors (finalize_tiles allocates them)
  if (cudaStreamSynchronize(s) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "set_obs_encoder: sync"));
  *out = st;
  return 0;
}

void enc_stage_destroy(EncStage* st) {
  if (!st) return;
  for (void* p : st->allocs) cudaFree(p);
  delete st;
}

int enc_stage_row_floats(const EncStage* st) { return st->RW; }

float* enc_stage_raw(EncStage* st, int which) { return st->raw[which]; }

int enc_stage_encode(EncStage* st, int which, const float* done, int n, int n_done, float* dst, cudaStream_t s) {
  const int nb = which ? n_done : n;
  if (nb < 1) return 0;
  if (int rc = set_batch(st->layers, st->groups[which], st->built_n[which], nb, st->allocs, s)) return rc;
  const int* map = nullptr;
  if (which) {
    enc_done_map<<<1, 32, 0, s>>>(done, n, st->map);
    map = st->map;
  }
  const EncLayer& y0 = st->layers[0];
  const int D = st->cfg.encoding_dim;
  if (st->precision == B2G_PREC_BF16X3) {
    if (int rc = tc_forward(st->layers, st->planes, st->groups[which], st->cfg, st->raw[which], st->RW, map, nb, dst, st->E,
                            st->num_sms, s))
      return rc;
  } else {
    const int blocks_in = (int)std::min<long long>(((long long)nb * st->RW + 255) / 256, 132 * 8);
    enc_stage_in<<<blocks_in, 256, 0, s>>>(st->raw[which], st->RW, map, nb, st->cfg.width, st->cfg.channels, y0.hp, y0.wp, y0.pad_t,
                                           y0.pad_l, y0.in, D, dst, st->E);
    for (auto& g : st->groups[which]) gg_simt_launch(g.dev, 1, g.total_tiles, s);
  }
  const int blocks_out = (int)std::min<long long>(((long long)nb * D + 255) / 256, 132 * 8);
  enc_stage_out<<<blocks_out, 256, 0, s>>>(st->z, st->zs, map, nb, D, dst, st->E);
  CK(cudaGetLastError());
  return 0;
}

}  // namespace b2g
