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

// map[j] = index of the j-th finished env (done[i] != 0), i < n
__global__ void enc_done_map(const float* __restrict__ done, int n, int* __restrict__ map) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  int j = 0;
  for (int i = 0; i < n; ++i)
    if (done[i] != 0.f) map[j++] = i;
}
}  // namespace

struct b2g_encoder {
  b2g_encoder_cfg cfg{};
  cudaStream_t stream = nullptr;
  std::vector<void*> allocs;
  std::vector<EncLayer> layers;          // convs then the dense layer
  float* stage_in = nullptr;             // [N, H, W, C] as received
  float* z = nullptr;                    // [N, zs]
  int zs = 0;
  std::vector<GemmGroup> groups;         // one launch per layer (each consumes the previous one's output)
  int built_n = -1;
  float* pin_in = nullptr;
  float* pin_out = nullptr;
};

namespace {
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
    if (int rc = finalize_tiles(groups[l], allocs, s)) return rc;
  }
  built_n = n;
  return 0;
}
}  // namespace

extern "C" {

int b2g_encoder_create(const b2g_encoder_cfg* cfg, b2g_encoder** out) {
  if (!cfg || !out) return b2g_fail(B2G_EINVAL, "null argument");
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
  if (int rc = check_device(cfg->device)) return rc;
  b2g_encoder* h = new b2g_encoder();
  h->cfg = *cfg;
  h->layers = layers;
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
  if ((rc = build_tables(h->layers, (int)N, h->cfg.alpha, h->z, h->zs, h->groups, h->allocs, h->stream))) return bail(rc);
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
  const size_t in_numel = (size_t)n * h->cfg.height * h->cfg.width * h->cfg.channels;
  memcpy(h->pin_in, imgs, in_numel * sizeof(float));
  CK(cudaMemcpyAsync(h->stage_in, h->pin_in, in_numel * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  const int blocks = (int)std::min<size_t>((in_numel + 255) / 256, 132 * 8);
  enc_pad_copy<<<blocks, 256, 0, h->stream>>>(h->stage_in, y0.in, n, h->cfg.height, h->cfg.width, h->cfg.channels, y0.hp, y0.wp,
                                              y0.pad_t, y0.pad_l);
  for (auto& g : h->groups) gg_simt_launch(g.dev, 1, g.total_tiles, h->stream);
  CK(cudaGetLastError());
  CK(cudaMemcpy2DAsync(h->pin_out, h->cfg.encoding_dim * sizeof(float), h->z, h->zs * sizeof(float),
                        h->cfg.encoding_dim * sizeof(float), n, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  memcpy(out, h->pin_out, (size_t)n * h->cfg.encoding_dim * sizeof(float));
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
  if ((rc = build_tables(st->layers, rows, st->cfg.alpha, st->z, st->zs, st->groups[0], st->allocs, s))) return bail(rc);
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
  const int blocks_in = (int)std::min<long long>(((long long)nb * st->RW + 255) / 256, 132 * 8);
  enc_stage_in<<<blocks_in, 256, 0, s>>>(st->raw[which], st->RW, map, nb, st->cfg.width, st->cfg.channels, y0.hp, y0.wp, y0.pad_t,
                                         y0.pad_l, y0.in, D, dst, st->E);
  for (auto& g : st->groups[which]) gg_simt_launch(g.dev, 1, g.total_tiles, s);
  const int blocks_out = (int)std::min<long long>(((long long)nb * D + 255) / 256, 132 * 8);
  enc_stage_out<<<blocks_out, 256, 0, s>>>(st->z, st->zs, map, nb, D, dst, st->E);
  CK(cudaGetLastError());
  return 0;
}

}  // namespace b2g
