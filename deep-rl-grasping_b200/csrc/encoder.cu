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
#include <cuda_runtime.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/b200grasp.h"
#include "common.cuh"
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
// Offset tables for the whole capacity; a call with n < max_batch uses the leading n * out_h * out_w rows.
int build_tables(b2g_encoder* h) {
  const int N = h->cfg.max_batch, L = (int)h->layers.size();
  h->groups.resize(L);
  for (int l = 0; l < L; ++l) {
    EncLayer& y = h->layers[l];
    const bool dense = y.k == 0;
    // where this layer's output lands: interior of the next layer's bordered input, or z
    float* out;
    int o_hp, o_wp, o_pt, o_pl, o_c;
    if (dense) { out = h->z; o_hp = o_wp = 1; o_pt = o_pl = 0; o_c = h->zs; }
    else {
      const EncLayer& nx = h->layers[l + 1];
      out = nx.in; o_hp = nx.hp; o_wp = nx.wp; o_pt = nx.pad_t; o_pl = nx.pad_l; o_c = y.f;
    }
    const int M = N * y.out_h * y.out_w, R = y.R();
    std::vector<int> aM, cM, aR, bR, bN, cN;
    enc_fwd_tables(y, N, o_hp, o_wp, o_pt, o_pl, o_c, aM, cM, aR, bR, bN, cN);
    GemmDesc d = gemm_desc(y.in, nullptr, nullptr, y.w, nullptr, nullptr, out, nullptr, nullptr, M, y.f, R, enc_fwd_flags(y));
    d.bias = y.b; d.alpha = h->cfg.alpha;
    if (int rc = upload_table(h->allocs, h->stream, aM, &d.aM)) return rc;
    if (int rc = upload_table(h->allocs, h->stream, aR, &d.aR)) return rc;
    if (int rc = upload_table(h->allocs, h->stream, bR, &d.bR)) return rc;
    if (int rc = upload_table(h->allocs, h->stream, bN, &d.bN)) return rc;
    if (int rc = upload_table(h->allocs, h->stream, cM, &d.cM)) return rc;
    if (int rc = upload_table(h->allocs, h->stream, cN, &d.cN)) return rc;
    GemmGroup& g = h->groups[l];
    g.name = dense ? "enc_dense" : "enc_conv" + std::to_string(l);
    g.host = {d};
    if (int rc = finalize_tiles(g, h->allocs, h->stream)) return rc;
  }
  h->built_n = N;
  return 0;
}

int set_batch(b2g_encoder* h, int n) {
  if (h->built_n == n) return 0;
  for (size_t l = 0; l < h->layers.size(); ++l) {
    const EncLayer& y = h->layers[l];
    h->groups[l].host[0].M = n * y.out_h * y.out_w;
    if (int rc = finalize_tiles(h->groups[l], h->allocs, h->stream)) return rc;
  }
  h->built_n = n;
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
  if ((rc = build_tables(h))) return bail(rc);
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
  if (int rc = set_batch(h, n)) return rc;
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
