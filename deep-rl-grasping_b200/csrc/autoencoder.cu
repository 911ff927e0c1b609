// libb200grasp: convolutional auto-encoder TRAINING -- SURVEY.md section 8 row a12 (encoders.py:40-61 train / test / predict).
//
// The whole Keras model (encoders.py:84-136) on one handle, in fp32 on the CUDA cores (or bf16x3, below).  One training step is
//   forward of the 2L+2 layers -> MSE seed -> backward (input gradient of every layer but the first conv, weight and bias
//   gradient of every layer) -> Keras Adam.
// Every conv and dense contraction runs on the gather-GEMM engine (gg_simt.cu) from offset tables; the encoder half's
// forward uses the encoder handle's tables (enc_tables.cuh).  Layout of the intermediate tensors (all NHWC):
//   * a conv's input lives in a zero-bordered buffer ('same' padding), as in encoder.cu.  Decoder convs read the nearest
//     upsampling of the previous output, materialised into that buffer by ae_upsample.
//   * the gradient of a conv's pre-activation lives in a zero buffer D with sample (oy, ox) at (oy*s + k-1, ox*s + k-1):
//     the input gradient is then the plain correlation dXb[py] = sum_ky' D[py + ky'] * W[k-1-ky'] (zero insertion for
//     stride s > 1).  A decoder conv's input gradient also sums each u x u upsampling block, which folds into the same
//     gather: R runs over (i, j, ky', kx', f).  The epilogue multiplies by the LeakyReLU derivative of the previous layer,
//     taken from the sign of its stored output (GG_EPI_LRELU_GRAD), and writes straight into that layer's D.
//   * weight gradients are split-R gather-GEMMs accumulated with atomics; the bias gradient is the engine's column sum.
//     These reductions run over every pixel of the batch and their terms largely cancel (conv1's by a factor of several
//     hundred), so the rounding of every sum upstream of them counts: every contraction sums its exact fp32 products in
//     double (gg_simt_launch_ext; the output conv's weight gradient likewise), and the weight gradients accumulate
//     into a double arena that is rounded to fp32 once per step.  Stored activations and gradients stay fp32.
// The one-filter output conv would waste 63 of 64 tile columns on the engine, so its forward (fused with the MSE seed and
// the bias gradient) and its weight gradient are direct-convolution kernels over 8x8 pixel tiles staged in shared memory.
// Its input gradient (N = filters_0) runs on the engine.
//
// Precision B2G_PREC_BF16X3 (b2g_autoencoder_create2) runs every contraction whose operands the wgmma engine's
// register-staged producer can read on that engine (gg_tc.cu, GG_ACC64 instantiations, x3 = 1): the producer gathers the same
// fp32 tensors through the same offset tables in 16-byte groups of 4 consecutive values, splits each value into BF16 hi + lo in
// registers and the tensor cores sum hi*hi + hi*lo + lo*hi in fp32.  That covers the forward of every conv but the first and
// of both dense layers (bias + LeakyReLU epilogue), every input gradient but the output conv's (LeakyReLU-derivative epilogue
// into the previous layer's D) and every weight and bias gradient but the first conv's and the output conv's.  A weight
// gradient's split-R partial sums (the tensor cores' fp32 accumulators over one split's r-range; the bias: each producer
// thread's fp32 running sum of D over its share of that range) are added into the double arena with double atomics.
// conv1's forward and weight gradient (one input channel) and the output conv's input gradient (one filter) have no 4-element
// groups along their reduction or output rows, so they stay on gg_simt, as do the output conv's direct kernels and Adam.
// Nothing is kept as planes in HBM: the weights change every step and each activation and gradient is read once or twice.
//
// Training epochs keep the dataset on the device: each step gathers its batch rows through the epoch's permutation and a
// device cursor, so one captured graph per batch size replays every step (the partial last batch has its own graph).
// Loss sums are kept in double and read once per epoch.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <map>
#include <string>
#include <vector>

#include "../../include/b200grasp.h"
#include "common.cuh"
#include "enc_tables.cuh"
#include "host.cuh"

using namespace b2g;

namespace {
constexpr int AE_TILE = 8;            // output conv: 8 x 8 pixel tiles
constexpr int AE_WG_OUT = 8;          // output conv weight gradient: outputs per thread (k*k*filters_0 <= 256 * 8)
constexpr int AE_MAX_SMEM = 96 * 1024;
constexpr float AE_B1 = 0.9f, AE_B2 = 0.999f, AE_EPS = 1e-7f;   // keras.optimizers.Adam defaults, K.epsilon()

enum AeKind { ENC_CONV, ENC_DENSE, DEC_DENSE, DEC_CONV, OUT_CONV };

struct AeLayer {
  AeKind kind;
  EncLayer g;              // geometry (dense: R() input features, f outputs)
  int up = 1;              // decoder conv: nearest upsampling of the previous output
  int map_h = 1, map_w = 1, map_c = 0;   // the layer's output seen as a map (dense: decoder Reshape / [1, 1, zs])
  float* in = nullptr;     // conv: bordered input [N, hp, wp, in_c]; dense: rows [N, in_ld]
  int in_ld = 0;
  float* act = nullptr;    // post-activation output when no bordered buffer holds it: decoder maps [N, map], z [N, zs]
  float* D = nullptr;      // gradient of the pre-activation (see the file comment)
  int dh = 1, dw = 1;
  size_t w_off = 0, b_off = 0;
  bool loaded = false;
  size_t d_off(int b, int oy, int ox) const {   // element offset of output (b, oy, ox), channel 0, inside D
    if (g.k == 0) return (size_t)b * dw;      // dense: dw = row stride
    return (((size_t)b * dh + oy * g.s + g.k - 1) * dw + ox * g.s + g.k - 1) * g.f;
  }
};

struct AeGemm {
  GemmDesc d;
  int m_per = 0, r_per = 0;  // M or R per sample (the other extent is fixed)
  bool wgrad = false;
  bool tc = false;           // bf16x3: runs on the wgmma engine
};

struct AePlan {
  std::vector<GemmGroup> g;  // one group per contraction, in the order of `gemms`
  cudaGraphExec_t train = nullptr;
};

// ---------------------------------------------------------------------------------------------------------------- kernels
// batch rows -> interior of the first conv's bordered input, and their targets -> T [n, HW]
__global__ void ae_gather(const float* __restrict__ src, const float* __restrict__ tgt, const int* __restrict__ order,
                          const long long* __restrict__ cursor, long long base, int n, int H, int W, float* __restrict__ X0, int hp,
                          int wp, int pt, int pl, float* __restrict__ T) {
  const int HW = H * W;
  const long long c0 = cursor ? *cursor : 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)n * HW; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / HW), p = (int)(i - (long long)b * HW);
    const long long row = order ? order[c0 + b] : base + b;
    const int y = p / W, x = p - y * W;
    X0[((long long)b * hp + y + pt) * wp + x + pl] = src[row * HW + p];
    T[i] = tgt[row * HW + p];
  }
}

// nearest upsampling of A [n, h, w, c] by u into the interior of a bordered [n, hp, wp, c] buffer (c % 4 == 0)
__global__ void ae_upsample(const float* __restrict__ A, int n, int h, int w, int c, int u, float* __restrict__ U, int hp, int wp,
                            int pt, int pl) {
  const int c4 = c >> 2, H = h * u, W = w * u;
  const long long total = (long long)n * H * W * c4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(i % c4);
    long long p = i / c4;
    const int x = (int)(p % W); p /= W;
    const int y = (int)(p % H);
    const int b = (int)(p / H);
    const float4 v = reinterpret_cast<const float4*>(A)[(((long long)b * h + y / u) * w + x / u) * c4 + q];
    reinterpret_cast<float4*>(U)[(((long long)b * hp + y + pt) * wp + x + pl) * c4 + q] = v;
  }
}

// Stages the (8 + k - 1)^2 input patch of tile (ty0, tx0) of sample b into Us (pixel stride cin + 1 against bank conflicts).
__device__ __forceinline__ void ae_stage_patch(const float* __restrict__ U, int b, int ty0, int tx0, int hp, int wp, int cin, int k,
                                               float* Us) {
  const int PW = AE_TILE + k - 1, CP = cin + 1;
  for (int i = threadIdx.x; i < PW * PW * cin; i += blockDim.x) {
    const int c = i % cin, px = (i / cin) % PW, py = i / (cin * PW);
    const int gy = ty0 + py, gx = tx0 + px;
    Us[(py * PW + px) * CP + c] = (gy < hp && gx < wp) ? U[(((long long)b * hp + gy) * wp + gx) * cin + c] : 0.f;
  }
}

// Output conv (one filter, stride 1) forward on 8x8 tiles, fused with the mean-squared-error seed:
//   Y = b + sum U*W;  sumsq += (Y - T)^2;  D(oy, ox) = scale * (Y - T);  gbias += sum D   (grad != 0)
__global__ void __launch_bounds__(256) ae_out_fwd(const float* __restrict__ U, int hp, int wp, int cin, int k,
                                                  const float* __restrict__ Wt, const float* __restrict__ bias, int H, int W,
                                                  const float* __restrict__ T, float* __restrict__ Y, float* __restrict__ D, int dh,
                                                  int dw, float scale, double* __restrict__ sumsq, double* __restrict__ gbias, int grad) {
  extern __shared__ float sm[];
  const int PW = AE_TILE + k - 1, CP = cin + 1, KK = k * k * cin;
  float* Ws = sm;
  float* Us = sm + KK;
  __shared__ float part[4][64];
  __shared__ double red_sq[2];
  __shared__ float red_g[2];
  const int tx_n = (W + AE_TILE - 1) / AE_TILE, ty_n = (H + AE_TILE - 1) / AE_TILE;
  const int b = blockIdx.x / (tx_n * ty_n), t = blockIdx.x % (tx_n * ty_n);
  const int ty0 = (t / tx_n) * AE_TILE, tx0 = (t % tx_n) * AE_TILE;
  for (int i = threadIdx.x; i < KK; i += blockDim.x) Ws[i] = Wt[i];
  ae_stage_patch(U, b, ty0, tx0, hp, wp, cin, k, Us);
  __syncthreads();
  const int p = threadIdx.x & 63, q = threadIdx.x >> 6, py = p >> 3, px = p & 7;
  float acc = 0.f;
  for (int ky = 0; ky < k; ++ky)
    for (int kx = 0; kx < k; ++kx) {
      const float* u = Us + ((py + ky) * PW + px + kx) * CP;
      const float* w = Ws + (ky * k + kx) * cin;
      for (int c = q; c < cin; c += 4) acc = fmaf(u[c], w[c], acc);
    }
  part[q][p] = acc;
  __syncthreads();
  if (threadIdx.x < 64) {
    const int oy = ty0 + py, ox = tx0 + px;
    double sq = 0.0;
    float g = 0.f;
    if (oy < H && ox < W) {
      const float y = ((part[0][p] + part[1][p]) + (part[2][p] + part[3][p])) + bias[0];
      const size_t o = ((size_t)b * H + oy) * W + ox;
      if (Y) Y[o] = y;
      const float diff = y - T[o];
      sq = (double)diff * diff;
      if (grad) {
        g = scale * diff;
        D[((size_t)b * dh + oy + k - 1) * dw + ox + k - 1] = g;
      }
    }
    for (int s = 16; s; s >>= 1) {
      sq += __shfl_xor_sync(0xffffffffu, sq, s);
      g += __shfl_xor_sync(0xffffffffu, g, s);
    }
    if ((threadIdx.x & 31) == 0) { red_sq[threadIdx.x >> 5] = sq; red_g[threadIdx.x >> 5] = g; }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    atomicAdd(sumsq, red_sq[0] + red_sq[1]);
    if (grad) atomicAdd(gbias, (double)red_g[0] + (double)red_g[1]);
  }
}

// Output conv weight gradient: gW[(ky, kx, c)] = sum over pixels of U(oy + ky, ox + kx, c) * D(oy, ox).  Blocks walk the
// 8x8 tiles of the batch, each thread owns up to AE_WG_OUT weights and adds them once at the end.
__global__ void __launch_bounds__(256) ae_out_wgrad(const float* __restrict__ U, int hp, int wp, int cin, int k, int H, int W, int n,
                                                    const float* __restrict__ D, int dh, int dw, double* __restrict__ gW) {
  extern __shared__ float sm[];
  const int PW = AE_TILE + k - 1, CP = cin + 1, KK = k * k * cin;
  float* Us = sm;
  __shared__ float Ds[64];
  const int tx_n = (W + AE_TILE - 1) / AE_TILE, ty_n = (H + AE_TILE - 1) / AE_TILE, tiles = n * tx_n * ty_n;
  int oo[AE_WG_OUT];
  double acc[AE_WG_OUT];
#pragma unroll
  for (int j = 0; j < AE_WG_OUT; ++j) {
    const int o = threadIdx.x + j * blockDim.x;
    acc[j] = 0.0;
    if (o < KK) {
      const int c = o % cin, kx = (o / cin) % k, ky = o / (cin * k);
      oo[j] = (ky * PW + kx) * CP + c;
    } else {
      oo[j] = -1;
    }
  }
  for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int b = t / (tx_n * ty_n), tt = t % (tx_n * ty_n);
    const int ty0 = (tt / tx_n) * AE_TILE, tx0 = (tt % tx_n) * AE_TILE;
    __syncthreads();
    ae_stage_patch(U, b, ty0, tx0, hp, wp, cin, k, Us);
    if (threadIdx.x < 64) {
      const int oy = ty0 + (threadIdx.x >> 3), ox = tx0 + (threadIdx.x & 7);
      Ds[threadIdx.x] = (oy < H && ox < W) ? D[((size_t)b * dh + oy + k - 1) * dw + ox + k - 1] : 0.f;
    }
    __syncthreads();
    for (int p = 0; p < 64; ++p) {
      const float dv = Ds[p];
      const int po = ((p >> 3) * PW + (p & 7)) * CP;
#pragma unroll
      for (int j = 0; j < AE_WG_OUT; ++j)
        if (oo[j] >= 0) acc[j] = fma((double)Us[po + oo[j]], (double)dv, acc[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < AE_WG_OUT; ++j)
    if (oo[j] >= 0) atomicAdd(gW + threadIdx.x + j * blockDim.x, acc[j]);
}

// gradient arena: double sums -> fp32
__global__ void ae_round_grads(const double* __restrict__ G64, float* __restrict__ G, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) G[i] = (float)G64[i];
}

// Keras Adam, step t = ++counters[0]:  lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t); also advances the batch cursor counters[1].
__global__ void ae_adam_prep(long long* counters, const float* lr, float* lr_t, int n) {
  const long long t = ++counters[0];
  counters[1] += n;
  *lr_t = (float)((double)*lr * sqrt(1.0 - pow((double)AE_B2, (double)t)) / (1.0 - pow((double)AE_B1, (double)t)));
}

__global__ void ae_adam(float4* __restrict__ P, float4* __restrict__ Mo, float4* __restrict__ Vo, const float4* __restrict__ G,
                        const float* __restrict__ lr_t, int n4) {
  const float lr = *lr_t;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
    const float4 g = G[i];
    float4 m = Mo[i], v = Vo[i], p = P[i];
    float* mp = &m.x; float* vp = &v.x; float* pp = &p.x;
    const float* gp = &g.x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      mp[j] = AE_B1 * mp[j] + (1.f - AE_B1) * gp[j];
      vp[j] = AE_B2 * vp[j] + (1.f - AE_B2) * (gp[j] * gp[j]);
      pp[j] = pp[j] - lr * mp[j] / (sqrtf(vp[j]) + AE_EPS);
    }
    Mo[i] = m; Vo[i] = v; P[i] = p;
  }
}
}  // namespace

struct b2g_autoencoder {
  b2g_encoder_cfg cfg{};
  int precision = B2G_PREC_FP32_SIMT;
  cudaStream_t stream = nullptr;
  int num_sms = 132;
  std::vector<void*> allocs;
  std::vector<AeLayer> L;
  int zs = 0;
  size_t n_par = 0;                                  // arena length (floats, multiple of 4)
  float *P = nullptr, *G = nullptr, *Mo = nullptr, *Vo = nullptr;
  double* G64 = nullptr;                             // gradient sums of the step (double), rounded into G
  float* T = nullptr;                                // targets of the batch [N, HW]
  float* Y = nullptr;                                // reconstructions [N, HW]
  float* stage_in = nullptr;                         // host batches [N, HW] (inputs, targets)
  float* stage_tg = nullptr;
  float* pin = nullptr;                              // pinned [N, HW]
  double* sumsq = nullptr;
  long long* counters = nullptr;                     // [0] Adam t, [1] batch cursor
  float* d_lr = nullptr;
  float* lr_t = nullptr;
  float cur_lr = -1.f;
  float* data = nullptr; float* data_tg = nullptr; int* order = nullptr;
  long long n_data = 0, data_cap = 0;
  std::vector<AeGemm> fwd_g, bwd_g;                  // contractions at max_batch, in issue order
  std::map<int, AePlan> plans;
  size_t out_smem_fwd = 0, out_smem_wg = 0;
  ColIds col_ids;                                    // bf16x3: column-table identities of the wgmma descriptors
};

namespace {
int ae_upload(b2g_autoencoder* h, const std::vector<int>& v, const int** out) { return upload_table(h->allocs, h->stream, v, out); }

// Registers one contraction: tables -> device, flags; extents per sample for the batch-size plans.
int add_gemm(b2g_autoencoder* h, std::vector<AeGemm>& list, const float* A, const float* B, float* C, int M, int N, int R, int flags,
             const std::vector<int>& aM, const std::vector<int>& aR, const std::vector<int>& bN, const std::vector<int>& bR,
             const std::vector<int>& cM, const std::vector<int>& cN, int m_per, int r_per, const float* bias = nullptr,
             const float* mask = nullptr, const std::vector<int>* kM = nullptr, const std::vector<int>* kN = nullptr,
             float* colsum = nullptr) {
  AeGemm e;
  e.d = gemm_desc(A, nullptr, nullptr, B, nullptr, nullptr, C, nullptr, nullptr, M, N, R, flags);
  e.d.bias = bias; e.d.mask = mask; e.d.colsum = colsum; e.d.alpha = h->cfg.alpha;
  e.m_per = m_per; e.r_per = r_per; e.wgrad = (flags & GG_EPI_ATOMIC) != 0;
  // GG_A_SCALAR marks the operands without 4-element groups (one channel / one filter): gg_simt only
  e.tc = h->precision == B2G_PREC_BF16X3 && !(flags & GG_A_SCALAR);
  std::map<const int*, std::vector<int>> host;       // the column-side tables, for gg_tc_columns
  auto* hc = e.tc ? &host : nullptr;
  if (int rc = ae_upload(h, aM, &e.d.aM)) return rc;
  if (int rc = ae_upload(h, aR, &e.d.aR)) return rc;
  if (int rc = ae_upload(h, bN, &e.d.bN)) return rc;
  if (int rc = ae_upload(h, bR, &e.d.bR)) return rc;
  if (int rc = upload_table(h->allocs, h->stream, cM, &e.d.cM, hc)) return rc;
  if (int rc = upload_table(h->allocs, h->stream, cN, &e.d.cN, hc)) return rc;
  if (kM) if (int rc = upload_table(h->allocs, h->stream, *kM, &e.d.kM, hc)) return rc;
  if (kN) if (int rc = upload_table(h->allocs, h->stream, *kN, &e.d.kN, hc)) return rc;
  if (e.tc) gg_tc_columns(e.d, host, h->col_ids);
  list.push_back(e);
  return 0;
}
}  // namespace

namespace {
// Where the LeakyReLU output of layer j - 1 at map position (b, y, x), channel 0, is stored, and where its pre-activation
// gradient goes: the interior of layer j's bordered input (encoder convs) or the compact decoder map, and D of layer j - 1.
void prev_offsets(const b2g_autoencoder* h, int j, int b, int y, int x, int* act, int* dst) {
  const AeLayer& cur = h->L[j];
  const AeLayer& pv = h->L[j - 1];
  const int c = pv.map_c;
  if (pv.kind == ENC_CONV) *act = (int)((((size_t)b * cur.g.hp + y + cur.g.pad_t) * cur.g.wp + x + cur.g.pad_l) * c);
  else *act = (int)((((size_t)b * pv.map_h + y) * pv.map_w + x) * c);
  if (pv.kind == DEC_DENSE) *dst = (int)((size_t)b * pv.dw + ((size_t)y * pv.map_w + x) * c);
  else *dst = (int)pv.d_off(b, y, x);
}

// Input gradient of conv layer j (u x u upsampling folded in), times the LeakyReLU derivative of layer j - 1, into D of j - 1.
int add_conv_dgrad(b2g_autoencoder* h, int j) {
  const int N = h->cfg.max_batch;
  const AeLayer& cur = h->L[j];
  const EncLayer& y = cur.g;
  const int u = cur.up, hq = y.in_h / u, wq = y.in_w / u, c = y.in_c, f = y.f, k = y.k;
  const int M = N * hq * wq, R = u * u * k * k * f;
  std::vector<int> aM(M), kM(M), cM(M), aR(R), bR(R), bN(c), cN(c);
  for (int b = 0; b < N; ++b)
    for (int yy = 0; yy < hq; ++yy)
      for (int xx = 0; xx < wq; ++xx) {
        const int m = (b * hq + yy) * wq + xx;
        aM[m] = (int)((((size_t)b * cur.dh + yy * u + y.pad_t) * cur.dw + xx * u + y.pad_l) * f);
        prev_offsets(h, j, b, yy, xx, &kM[m], &cM[m]);
      }
  for (int i = 0; i < u; ++i)
    for (int jj = 0; jj < u; ++jj)
      for (int ky = 0; ky < k; ++ky)
        for (int kx = 0; kx < k; ++kx)
          for (int fi = 0; fi < f; ++fi) {
            const int r = (((i * u + jj) * k + ky) * k + kx) * f + fi;
            aR[r] = ((i + ky) * cur.dw + jj + kx) * f + fi;
            bR[r] = ((k - 1 - ky) * k + (k - 1 - kx)) * c * y.fs + fi;
          }
  for (int cc = 0; cc < c; ++cc) { bN[cc] = cc * y.fs; cN[cc] = cc; }
  const float* mask = h->L[j - 1].kind == ENC_CONV ? cur.in : h->L[j - 1].act;
  const int flags = GG_A_RVEC | GG_EPI_LRELU_GRAD | ((f & 3) ? GG_A_SCALAR : GG_B_RVEC);
  return add_gemm(h, h->bwd_g, cur.D, h->P + cur.w_off, h->L[j - 1].D, M, c, R, flags, aM, aR, bN, bR, cM, cN, hq * wq, 0, nullptr,
                  mask, &kM, &cN);
}

// Weight and bias gradient of conv layer j: M = (ky, kx, c), N = filters, R = (b, oy, ox) split across CTAs.
int add_conv_wgrad(b2g_autoencoder* h, int j) {
  const int N = h->cfg.max_batch;
  const AeLayer& cur = h->L[j];
  const EncLayer& y = cur.g;
  const int M = y.k * y.k * y.in_c, P = y.out_h * y.out_w, R = N * P;
  std::vector<int> aM(M), cM(M), aR(R), bR(R), bN(y.f), cN(y.f);
  for (int m = 0; m < M; ++m) {
    const int c = m % y.in_c, kx = (m / y.in_c) % y.k, ky = m / (y.in_c * y.k);
    aM[m] = (ky * y.wp + kx) * y.in_c + c;
    cM[m] = m * y.fs;
  }
  for (int b = 0; b < N; ++b)
    for (int oy = 0; oy < y.out_h; ++oy)
      for (int ox = 0; ox < y.out_w; ++ox) {
        const int r = (b * y.out_h + oy) * y.out_w + ox;
        aR[r] = (int)((((size_t)b * y.hp + oy * y.s) * y.wp + ox * y.s) * y.in_c);
        bR[r] = (int)cur.d_off(b, oy, ox);
      }
  for (int n = 0; n < y.f; ++n) bN[n] = cN[n] = n;
  return add_gemm(h, h->bwd_g, cur.in, cur.D, reinterpret_cast<float*>(h->G64 + cur.w_off), M, y.f, R,
                  GG_EPI_ATOMIC | GG_COLSUM | ((y.in_c & 3) ? GG_A_SCALAR : 0), aM, aR, bN, bR, cM, cN, 0, P, nullptr, nullptr,
                  nullptr, nullptr, reinterpret_cast<float*>(h->G64 + cur.b_off));
}

// Weight and bias gradient of a dense layer: M = input features, N = outputs, R = batch.
int add_dense_wgrad(b2g_autoencoder* h, int j) {
  const int N = h->cfg.max_batch;
  const AeLayer& cur = h->L[j];
  const int M = cur.g.R(), F = cur.g.f;
  std::vector<int> aM = iota_tab(M), aR = iota_tab(N, cur.in_ld), bN = iota_tab(F), bR = iota_tab(N, cur.dw), cM = iota_tab(M, cur.g.fs);
  return add_gemm(h, h->bwd_g, cur.in, cur.D, reinterpret_cast<float*>(h->G64 + cur.w_off), M, F, N, GG_EPI_ATOMIC | GG_COLSUM, aM,
                  aR, bN, bR, cM, bN, 0, 1, nullptr, nullptr, nullptr, nullptr, reinterpret_cast<float*>(h->G64 + cur.b_off));
}

// Input gradient of a dense layer times the LeakyReLU derivative of its input: decoder dense -> z, encoder dense -> last conv.
int add_dense_dgrad(b2g_autoencoder* h, int j) {
  const int N = h->cfg.max_batch;
  const AeLayer& cur = h->L[j];
  const AeLayer& pv = h->L[j - 1];
  const int Rin = cur.g.R(), F = cur.g.f;
  std::vector<int> aM = iota_tab(N, cur.dw), aR = iota_tab(F), bN = iota_tab(Rin, cur.g.fs), bR = iota_tab(F), kM = iota_tab(N, cur.in_ld),
                   kN = iota_tab(Rin), cM(N), cN(Rin);
  for (int b = 0; b < N; ++b) cM[b] = (int)(pv.kind == ENC_DENSE ? (size_t)b * pv.dw : (size_t)b * pv.dh * pv.dw * pv.g.f);
  for (int r = 0; r < Rin; ++r) {
    if (pv.kind == ENC_DENSE) cN[r] = r;
    else {
      const int c = r % pv.g.f, x = (r / pv.g.f) % pv.g.out_w, y = r / (pv.g.f * pv.g.out_w);
      cN[r] = (int)pv.d_off(0, y, x) + c;
    }
  }
  const float* mask = pv.kind == ENC_DENSE ? pv.act : cur.in;
  return add_gemm(h, h->bwd_g, cur.D, h->P + cur.w_off, pv.D, N, Rin, F, GG_A_RVEC | GG_B_RVEC | GG_EPI_LRELU_GRAD, aM, aR, bN, bR,
                  cM, cN, 1, 0, nullptr, mask, &kM, &kN);
}

int build(b2g_autoencoder* h) {
  const int N = h->cfg.max_batch, Lc = h->cfg.n_layers, nL = (int)h->L.size();
  // ---- forward: encoder convs + encoder dense (encoder.cu's tables), decoder dense, decoder convs
  for (int l = 0; l <= Lc; ++l) {
    const AeLayer& cur = h->L[l];
    const EncLayer& y = cur.g;
    float* out;
    int o_hp, o_wp, o_pt, o_pl, o_c;
    if (l == Lc) { out = cur.act; o_hp = o_wp = 1; o_pt = o_pl = 0; o_c = h->zs; }
    else {
      const EncLayer& nx = h->L[l + 1].g;
      out = h->L[l + 1].in; o_hp = nx.hp; o_wp = nx.wp; o_pt = nx.pad_t; o_pl = nx.pad_l; o_c = y.f;
    }
    std::vector<int> aM, cM, aR, bR, bN, cN;
    enc_fwd_tables(y, N, o_hp, o_wp, o_pt, o_pl, o_c, aM, cM, aR, bR, bN, cN);
    if (int rc = add_gemm(h, h->fwd_g, cur.in, h->P + cur.w_off, out, N * y.out_h * y.out_w, y.f, y.R(), enc_fwd_flags(y), aM, aR, bN,
                          bR, cM, cN, y.out_h * y.out_w, 0, h->P + cur.b_off))
      return rc;
  }
  {
    const AeLayer& dd = h->L[Lc + 1];
    const int R = dd.g.R(), F = dd.g.f;
    std::vector<int> aM = iota_tab(N, h->zs), aR = iota_tab(R), bN = iota_tab(F), bR = iota_tab(R, dd.g.fs), cM = iota_tab(N, F);
    if (int rc = add_gemm(h, h->fwd_g, dd.in, h->P + dd.w_off, dd.act, N, F, R, GG_A_RVEC | GG_EPI_BIAS_LRELU, aM, aR, bN, bR, cM, bN, 1,
                          0, h->P + dd.b_off))
      return rc;
  }
  for (int j = Lc + 2; j < nL - 1; ++j) {
    const AeLayer& cur = h->L[j];
    const EncLayer& y = cur.g;
    std::vector<int> aM, cM, aR, bR, bN, cN;
    enc_fwd_tables(y, N, y.out_h, y.out_w, 0, 0, y.f, aM, cM, aR, bR, bN, cN);
    if (int rc = add_gemm(h, h->fwd_g, cur.in, h->P + cur.w_off, cur.act, N * y.out_h * y.out_w, y.f, y.R(), enc_fwd_flags(y), aM, aR,
                          bN, bR, cM, cN, y.out_h * y.out_w, 0, h->P + cur.b_off))
      return rc;
  }
  // ---- backward, in issue order (the output conv's weight gradient is a kernel of its own)
  for (int j = nL - 1; j >= 0; --j) {
    const AeKind kd = h->L[j].kind;
    int rc = 0;
    if (kd == ENC_CONV || kd == DEC_CONV) rc = add_conv_wgrad(h, j);
    else if (kd == ENC_DENSE || kd == DEC_DENSE) rc = add_dense_wgrad(h, j);
    if (rc) return rc;
    if (j == 0) break;
    rc = (kd == ENC_DENSE || kd == DEC_DENSE) ? add_dense_dgrad(h, j) : add_conv_dgrad(h, j);
    if (rc) return rc;
  }
  return 0;
}

int get_plan(b2g_autoencoder* h, int n, AePlan** out) {
  auto it = h->plans.find(n);
  if (it != h->plans.end()) { *out = &it->second; return 0; }
  AePlan p;
  for (const auto* list : {&h->fwd_g, &h->bwd_g})
    for (const AeGemm& e : *list) {
      GemmGroup g;
      g.name = "ae";
      GemmDesc d = e.d;
      if (e.m_per) d.M = e.m_per * n;
      if (e.r_per) d.R = e.r_per * n;
      if (e.tc) {
        // persistent grid of min(tiles, SMs) CTAs: a weight gradient splits R so that its tiles fill the SMs once
        d.tiles_m = (d.M + GG_TC_BM - 1) / GG_TC_BM;
        d.tiles_n = (d.N + GG_TC_BN - 1) / GG_TC_BN;
        if (e.wgrad) d.splitR = std::max(1, std::min(h->num_sms / (d.tiles_m * d.tiles_n), d.R / 512));
        d.tile_start = 0;
        d.tile_count = d.tiles_m * d.tiles_n * d.splitR;
        g.host = {d};
        g.total_tiles = d.tile_count;
        g.tc = true;
        p.g.push_back(g);
        continue;
      }
      if (e.wgrad) {
        const int tiles = ((d.M + GG_SIMT_BM - 1) / GG_SIMT_BM) * ((d.N + GG_SIMT_BN - 1) / GG_SIMT_BN);
        d.splitR = std::max(1, std::min((2 * h->num_sms + tiles - 1) / tiles, d.R / 256));
      }
      g.host = {d};
      if (int rc = finalize_tiles(g, h->allocs, h->stream)) return rc;
      p.g.push_back(g);
    }
  *out = &(h->plans[n] = p);
  return 0;
}

// one contraction: gg_tc (GG_ACC64, x3 = 1) or gg_simt_launch_ext; a failed launch shows in cudaGetLastError
void launch_group(b2g_autoencoder* h, const GemmGroup& g) {
  if (!g.tc) { gg_simt_launch_ext(g.dev, 1, g.total_tiles, h->stream); return; }
  const GemmDesc& d = g.host[0];
  gg_tc_launch(g.host.data(), 1, g.total_tiles, (d.flags & (GG_A_RVEC | GG_B_RVEC)) | GG_ACC64, 1, h->num_sms, h->stream);
}

int grid_for(long long work) { return (int)std::max<long long>(1, std::min<long long>((work + 255) / 256, 132 * 8)); }

// gather (batch rows -> first conv input, targets -> T) from src / tgt through order[cursor + b], or rows base + b
void issue_gather(b2g_autoencoder* h, int n, const float* src, const float* tgt, const int* order, const long long* cursor,
                  long long base) {
  const AeLayer& l0 = h->L[0];
  ae_gather<<<grid_for((long long)n * h->cfg.height * h->cfg.width), 256, 0, h->stream>>>(
      src, tgt, order, cursor, base, n, h->cfg.height, h->cfg.width, l0.in, l0.g.hp, l0.g.wp, l0.g.pad_t, l0.g.pad_l, h->T);
}

void issue_forward(b2g_autoencoder* h, AePlan& p, int n, bool grad, float* Y) {
  const int Lc = h->cfg.n_layers, nL = (int)h->L.size();
  int k = 0;
  for (int l = 0; l <= Lc + 1; ++l) launch_group(h, p.g[k++]);
  for (int j = Lc + 2; j < nL; ++j) {
    const AeLayer& pv = h->L[j - 1];
    const AeLayer& cur = h->L[j];
    ae_upsample<<<grid_for((long long)n * cur.g.in_h * cur.g.in_w * pv.map_c / 4), 256, 0, h->stream>>>(
        pv.act, n, pv.map_h, pv.map_w, pv.map_c, cur.up, cur.in, cur.g.hp, cur.g.wp, cur.g.pad_t, cur.g.pad_l);
    if (cur.kind == DEC_CONV) {
      launch_group(h, p.g[k++]);
    } else {
      const int H = h->cfg.height, W = h->cfg.width;
      const int tiles = ((H + AE_TILE - 1) / AE_TILE) * ((W + AE_TILE - 1) / AE_TILE);
      ae_out_fwd<<<n * tiles, 256, h->out_smem_fwd, h->stream>>>(cur.in, cur.g.hp, cur.g.wp, cur.g.in_c, cur.g.k, h->P + cur.w_off,
                                                                 h->P + cur.b_off, H, W, h->T, Y, cur.D, cur.dh, cur.dw,
                                                                 2.f / ((float)n * H * W), h->sumsq, h->G64 + cur.b_off, grad ? 1 : 0);
    }
  }
}

void issue_backward(b2g_autoencoder* h, AePlan& p, int n) {
  const AeLayer& o = h->L.back();
  const int H = h->cfg.height, W = h->cfg.width;
  const int tiles = n * ((H + AE_TILE - 1) / AE_TILE) * ((W + AE_TILE - 1) / AE_TILE);
  ae_out_wgrad<<<std::min(tiles, 2 * h->num_sms), 256, h->out_smem_wg, h->stream>>>(o.in, o.g.hp, o.g.wp, o.g.in_c, o.g.k, H, W, n, o.D,
                                                                                   o.dh, o.dw, h->G64 + o.w_off);
  for (size_t k = h->fwd_g.size(); k < p.g.size(); ++k) launch_group(h, p.g[k]);
  ae_round_grads<<<grid_for((long long)h->n_par), 256, 0, h->stream>>>(h->G64, h->G, (int)h->n_par);
}

void issue_adam(b2g_autoencoder* h, int n) {
  ae_adam_prep<<<1, 1, 0, h->stream>>>(h->counters, h->d_lr, h->lr_t, n);
  const int n4 = (int)(h->n_par / 4);
  ae_adam<<<grid_for(n4), 256, 0, h->stream>>>((float4*)h->P, (float4*)h->Mo, (float4*)h->Vo, (const float4*)h->G, h->lr_t, n4);
}

// One training step on the batch that issue_gather staged (or gathers it from the dataset when from_data).
int issue_step(b2g_autoencoder* h, AePlan& p, int n, bool from_data, bool apply) {
  CK(cudaMemsetAsync(h->G64, 0, h->n_par * sizeof(double), h->stream));
  if (from_data) issue_gather(h, n, h->data, h->data_tg ? h->data_tg : h->data, h->order, h->counters + 1, 0);
  issue_forward(h, p, n, true, nullptr);
  issue_backward(h, p, n);
  if (apply) issue_adam(h, n);
  CK(cudaGetLastError());
  return 0;
}

int check_layer(const b2g_autoencoder* h, int layer, size_t kn, size_t bn) {
  if (!h) return b2g_fail(B2G_EINVAL, "null handle");
  if (layer < 0 || layer >= (int)h->L.size()) return b2g_fail(B2G_EINVAL, "layer out of range");
  const EncLayer& y = h->L[layer].g;
  if (kn != (size_t)y.R() * y.f || bn != (size_t)y.f)
    return b2g_fail(B2G_EINVAL, "layer " + std::to_string(layer) + ": expected kernel numel " + std::to_string((size_t)y.R() * y.f) +
                                    ", bias numel " + std::to_string(y.f));
  return 0;
}

int copy_out(b2g_autoencoder* h, const float* arena, int layer, float* kernel, float* bias) {
  const AeLayer& y = h->L[layer];
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemcpy2DAsync(kernel, y.g.f * sizeof(float), arena + y.w_off, y.g.fs * sizeof(float), y.g.f * sizeof(float), y.g.R(),
                        cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(bias, arena + y.b_off, y.g.f * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}

int need_weights(const b2g_autoencoder* h) {
  for (size_t l = 0; l < h->L.size(); ++l)
    if (!h->L[l].loaded) return b2g_fail(B2G_ESTATE, "auto-encoder layer " + std::to_string(l) + " has no weights");
  return 0;
}

// host images [n, HW] -> staging (and targets) -> first conv input
int stage_batch(b2g_autoencoder* h, const float* in, const float* tg, int n) {
  const size_t bytes = (size_t)n * h->cfg.height * h->cfg.width * sizeof(float);
  memcpy(h->pin, in, bytes);
  CK(cudaMemcpyAsync(h->stage_in, h->pin, bytes, cudaMemcpyHostToDevice, h->stream));
  if (tg) {
    CK(cudaStreamSynchronize(h->stream));
    memcpy(h->pin, tg, bytes);
    CK(cudaMemcpyAsync(h->stage_tg, h->pin, bytes, cudaMemcpyHostToDevice, h->stream));
  }
  issue_gather(h, n, h->stage_in, tg ? h->stage_tg : h->stage_in, nullptr, nullptr, 0);
  return 0;
}
}  // namespace

extern "C" {

int b2g_autoencoder_create(const b2g_encoder_cfg* cfg, b2g_autoencoder** out) {
  return b2g_autoencoder_create2(cfg, B2G_PREC_FP32_SIMT, out);
}

int b2g_autoencoder_create2(const b2g_encoder_cfg* cfg, int32_t precision, b2g_autoencoder** out) {
  if (!cfg || !out) return b2g_fail(B2G_EINVAL, "null argument");
  if (precision == B2G_PREC_BF16)
    return b2g_fail(B2G_EINVAL, "auto-encoder precision B2G_PREC_BF16: single-pass BF16 training is not offered; use "
                                "B2G_PREC_FP32_SIMT or B2G_PREC_BF16X3");
  if (precision != B2G_PREC_FP32_SIMT && precision != B2G_PREC_BF16X3)
    return b2g_fail(B2G_EINVAL, "auto-encoder precision " + std::to_string(precision) +
                                    ": expected B2G_PREC_FP32_SIMT (0) or B2G_PREC_BF16X3 (1)");
  if (cfg->n_layers < 1 || cfg->n_layers > B2G_ENC_MAX_LAYERS) return b2g_fail(B2G_EINVAL, "n_layers out of range");
  if (cfg->height < 1 || cfg->width < 1 || cfg->encoding_dim < 1 || cfg->max_batch < 1)
    return b2g_fail(B2G_EINVAL, "non-positive dimension");
  // The backward takes the LeakyReLU derivative from the sign of the stored output; with alpha < 0 a negative
  // pre-activation stores a positive value, so its derivative would come out as 1 instead of alpha.
  if (!(cfg->alpha >= 0.f) || !std::isfinite(cfg->alpha))
    return b2g_fail(B2G_EINVAL, "the auto-encoder trains with alpha >= 0 only (alpha = " + std::to_string(cfg->alpha) +
                                    "): its backward reads the LeakyReLU derivative from the sign of the stored output");
  if (cfg->channels != 1) return b2g_fail(B2G_EINVAL, "the auto-encoder reconstructs one-channel images (channels must be 1)");
  for (int l = 0; l < cfg->n_layers; ++l)
    if (cfg->filters[l] < 1 || (cfg->filters[l] & 3)) return b2g_fail(B2G_EINVAL, "auto-encoder filters must be multiples of 4");
  std::vector<EncLayer> enc;
  if (int rc = enc_geometry(*cfg, enc)) return rc;
  const int Lc = cfg->n_layers;
  std::vector<AeLayer> L;
  for (int l = 0; l <= Lc; ++l) {
    AeLayer a;
    a.kind = l < Lc ? ENC_CONV : ENC_DENSE;
    a.g = enc[l];
    if (l < Lc) { a.map_h = a.g.out_h; a.map_w = a.g.out_w; a.map_c = a.g.f; }
    else { a.map_c = a.g.fs; }
    L.push_back(a);
  }
  const int hL = enc[Lc].in_h, wL = enc[Lc].in_w, cL = enc[Lc].in_c;
  {
    AeLayer a;
    a.kind = DEC_DENSE;
    EncLayer& g = a.g;
    g.in_h = g.in_w = 1; g.in_c = cfg->encoding_dim; g.k = g.s = 0; g.f = hL * wL * cL; g.fs = g.f; g.out_h = g.out_w = 1;
    g.hp = g.wp = 1;
    a.map_h = hL; a.map_w = wL; a.map_c = cL;
    L.push_back(a);
  }
  int hq = hL, wq = wL, cq = cL;
  for (int i = Lc - 1; i >= 0; --i) {
    AeLayer a;
    a.kind = i > 0 ? DEC_CONV : OUT_CONV;
    a.up = cfg->strides[i];
    a.g = enc_conv_layer(hq * a.up, wq * a.up, cq, cfg->kernel[i], 1, i > 0 ? cfg->filters[i - 1] : 1);
    if (i == 0) a.g.fs = 1;
    a.map_h = a.g.out_h; a.map_w = a.g.out_w; a.map_c = a.g.f;
    hq = a.g.out_h; wq = a.g.out_w; cq = a.g.f;
    L.push_back(a);
  }
  if (hq != cfg->height || wq != cfg->width)
    return b2g_fail(B2G_EINVAL, "the decoder returns " + std::to_string(hq) + "x" + std::to_string(wq) + " instead of " +
                                    std::to_string(cfg->height) + "x" + std::to_string(cfg->width) + " (strides do not invert)");
  const EncLayer& og = L.back().g;
  const int PW = AE_TILE + og.k - 1;
  const size_t smem_fwd = ((size_t)og.k * og.k * og.in_c + (size_t)PW * PW * (og.in_c + 1)) * sizeof(float);
  const size_t smem_wg = (size_t)PW * PW * (og.in_c + 1) * sizeof(float);
  if ((size_t)og.k * og.k * og.in_c > 256 * AE_WG_OUT)
    return b2g_fail(B2G_EINVAL, "output conv too large: kernel_0^2 * filters_0 = " + std::to_string(og.k * og.k * og.in_c) +
                                    " must be <= 2048");
  if (smem_fwd > AE_MAX_SMEM)
    return b2g_fail(B2G_EINVAL, "output conv too large: its forward needs " + std::to_string(smem_fwd) +
                                    " B of shared memory ((kernel_0^2 * filters_0 + (kernel_0 + 7)^2 * (filters_0 + 1)) * 4), "
                                    "more than 98304");
  if (int rc = check_device(cfg->device)) return rc;

  b2g_autoencoder* h = new b2g_autoencoder();
  h->cfg = *cfg;
  h->precision = precision;
  h->L = L;
  h->out_smem_fwd = smem_fwd; h->out_smem_wg = smem_wg;
  auto bail = [&](int rc) { b2g_autoencoder_destroy(h); return rc; };
  if (int rc = check_device(cfg->device, &h->num_sms)) return bail(rc);
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "stream create"));
  const size_t N = cfg->max_batch;
  const int HW = cfg->height * cfg->width;
  h->zs = enc[Lc].fs;
  // arena offsets
  size_t off = 0;
  for (auto& y : h->L) {
    y.w_off = off; off += ((size_t)y.g.R() * y.g.fs + 3) / 4 * 4;
    y.b_off = off; off += ((size_t)y.g.fs + 3) / 4 * 4;
  }
  h->n_par = off;
  int rc;
  size_t biggest = 0;
  for (auto& y : h->L) {
    if (y.kind == ENC_CONV || y.kind == DEC_CONV || y.kind == OUT_CONV) {
      y.dh = y.g.in_h + y.g.pad_t + y.g.k - 1;
      y.dw = y.g.in_w + y.g.pad_l + y.g.k - 1;
      biggest = std::max({biggest, N * y.g.hp * y.g.wp * y.g.in_c, N * y.dh * y.dw * y.g.f});
    } else {
      y.dh = 1; y.dw = y.g.fs;
    }
  }
  if (biggest > (size_t)((1u << 31) - 1)) return bail(b2g_fail(B2G_EINVAL, "max_batch too large for 32-bit offset tables"));
  for (int l = 0; l < (int)h->L.size(); ++l) {
    AeLayer& y = h->L[l];
    switch (y.kind) {
      case ENC_CONV: case DEC_CONV: case OUT_CONV:
        if ((rc = dev_alloc(h->allocs, h->stream, &y.in, N * y.g.hp * y.g.wp * y.g.in_c))) return bail(rc);
        if ((rc = dev_alloc(h->allocs, h->stream, &y.D, N * y.dh * y.dw * y.g.f))) return bail(rc);
        if (y.kind == DEC_CONV && (rc = dev_alloc(h->allocs, h->stream, &y.act, N * y.g.out_h * y.g.out_w * y.g.f))) return bail(rc);
        break;
      case ENC_DENSE:
        y.in_ld = y.g.R();
        if ((rc = dev_alloc(h->allocs, h->stream, &y.in, N * y.in_ld))) return bail(rc);
        if ((rc = dev_alloc(h->allocs, h->stream, &y.act, N * h->zs))) return bail(rc);
        if ((rc = dev_alloc(h->allocs, h->stream, &y.D, N * h->zs))) return bail(rc);
        break;
      case DEC_DENSE:
        y.in = h->L[l - 1].act; y.in_ld = h->zs;
        if ((rc = dev_alloc(h->allocs, h->stream, &y.act, N * y.g.f))) return bail(rc);
        if ((rc = dev_alloc(h->allocs, h->stream, &y.D, N * y.g.f))) return bail(rc);
        break;
    }
  }
  if ((rc = dev_alloc(h->allocs, h->stream, &h->P, h->n_par)) || (rc = dev_alloc(h->allocs, h->stream, &h->G, h->n_par)) ||
      (rc = dev_alloc(h->allocs, h->stream, &h->G64, h->n_par)) || (rc = dev_alloc(h->allocs, h->stream, &h->Mo, h->n_par)) || (rc = dev_alloc(h->allocs, h->stream, &h->Vo, h->n_par)) ||
      (rc = dev_alloc(h->allocs, h->stream, &h->T, N * HW)) || (rc = dev_alloc(h->allocs, h->stream, &h->Y, N * HW)) ||
      (rc = dev_alloc(h->allocs, h->stream, &h->stage_in, N * HW)) || (rc = dev_alloc(h->allocs, h->stream, &h->stage_tg, N * HW)) ||
      (rc = dev_alloc(h->allocs, h->stream, &h->sumsq, 1)) || (rc = dev_alloc(h->allocs, h->stream, &h->counters, 2)) ||
      (rc = dev_alloc(h->allocs, h->stream, &h->d_lr, 1)) || (rc = dev_alloc(h->allocs, h->stream, &h->lr_t, 1)))
    return bail(rc);
  if (cudaMallocHost(&h->pin, N * HW * sizeof(float)) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "pinned staging allocation failed"));
  if (smem_fwd > 48 * 1024 && cudaFuncSetAttribute(ae_out_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_fwd) != cudaSuccess)
    return bail(b2g_fail(B2G_ECUDA, "output conv shared memory"));
  if (smem_wg > 48 * 1024 && cudaFuncSetAttribute(ae_out_wgrad, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_wg) != cudaSuccess)
    return bail(b2g_fail(B2G_ECUDA, "output conv shared memory"));
  if (precision == B2G_PREC_BF16X3 && gg_tc_acc64_init() != cudaSuccess)
    return bail(b2g_fail(B2G_ECUDA, "wgmma engine shared memory"));
  if ((rc = build(h))) return bail(rc);
  if (cudaStreamSynchronize(h->stream) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "auto-encoder create sync"));
  *out = h;
  return 0;
}

int b2g_autoencoder_destroy(b2g_autoencoder* h) {
  if (!h) return 0;
  cudaSetDevice(h->cfg.device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (auto& kv : h->plans)
    if (kv.second.train) cudaGraphExecDestroy(kv.second.train);
  for (void* p : h->allocs) cudaFree(p);
  if (h->data) cudaFree(h->data);
  if (h->data_tg) cudaFree(h->data_tg);
  if (h->order) cudaFree(h->order);
  if (h->pin) cudaFreeHost(h->pin);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

int b2g_autoencoder_n_layers(const b2g_autoencoder* h) { return h ? (int)h->L.size() : -1; }

int b2g_autoencoder_layer_shape(const b2g_autoencoder* h, int layer, int64_t* kernel_numel, int64_t* bias_numel) {
  if (!h || layer < 0 || layer >= (int)h->L.size()) return b2g_fail(B2G_EINVAL, "layer out of range");
  const EncLayer& y = h->L[layer].g;
  if (kernel_numel) *kernel_numel = (int64_t)y.R() * y.f;
  if (bias_numel) *bias_numel = y.f;
  return 0;
}

int b2g_autoencoder_set_weights(b2g_autoencoder* h, int layer, const float* kernel, size_t kernel_numel, const float* bias,
                                size_t bias_numel) {
  if (!kernel || !bias) return b2g_fail(B2G_EINVAL, "null argument");
  if (int rc = check_layer(h, layer, kernel_numel, bias_numel)) return rc;
  AeLayer& y = h->L[layer];
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemcpy2DAsync(h->P + y.w_off, y.g.fs * sizeof(float), kernel, y.g.f * sizeof(float), y.g.f * sizeof(float), y.g.R(),
                        cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(h->P + y.b_off, bias, y.g.f * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  y.loaded = true;
  return 0;
}

int b2g_autoencoder_get_weights(b2g_autoencoder* h, int layer, float* kernel, size_t kernel_numel, float* bias, size_t bias_numel) {
  if (!kernel || !bias) return b2g_fail(B2G_EINVAL, "null argument");
  if (int rc = check_layer(h, layer, kernel_numel, bias_numel)) return rc;
  if (!h->L[layer].loaded) return b2g_fail(B2G_ESTATE, "auto-encoder layer " + std::to_string(layer) + " has no weights");
  return copy_out(h, h->P, layer, kernel, bias);
}

int b2g_autoencoder_get_grad(b2g_autoencoder* h, int layer, float* kernel, size_t kernel_numel, float* bias, size_t bias_numel) {
  if (!kernel || !bias) return b2g_fail(B2G_EINVAL, "null argument");
  if (int rc = check_layer(h, layer, kernel_numel, bias_numel)) return rc;
  return copy_out(h, h->G, layer, kernel, bias);
}

int b2g_autoencoder_reset_optimizer(b2g_autoencoder* h) {
  if (!h) return b2g_fail(B2G_EINVAL, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemsetAsync(h->Mo, 0, h->n_par * sizeof(float), h->stream));
  CK(cudaMemsetAsync(h->Vo, 0, h->n_par * sizeof(float), h->stream));
  CK(cudaMemsetAsync(h->counters, 0, 2 * sizeof(long long), h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}

int b2g_autoencoder_set_dataset(b2g_autoencoder* h, const float* inputs, const float* targets, int64_t n) {
  if (!h || !inputs || n < 1) return b2g_fail(B2G_EINVAL, "null argument or empty dataset");
  CK(cudaSetDevice(h->cfg.device));
  const size_t HW = (size_t)h->cfg.height * h->cfg.width;
  CK(cudaStreamSynchronize(h->stream));
  const bool grow = n > h->data_cap || (targets && !h->data_tg);
  if (grow) {     // graphs captured the old buffers
    for (auto& kv : h->plans)
      if (kv.second.train) { cudaGraphExecDestroy(kv.second.train); kv.second.train = nullptr; }
    const long long cap = std::max<long long>(n, h->data_cap);
    if (h->data) { cudaFree(h->data); h->data = nullptr; }
    if (h->data_tg) { cudaFree(h->data_tg); h->data_tg = nullptr; }
    if (h->order) { cudaFree(h->order); h->order = nullptr; }
    CK(cudaMalloc(&h->data, cap * HW * sizeof(float)));
    if (targets) CK(cudaMalloc(&h->data_tg, cap * HW * sizeof(float)));
    CK(cudaMalloc(&h->order, cap * sizeof(int)));
    h->data_cap = cap;
  }
  CK(cudaMemcpy(h->data, inputs, n * HW * sizeof(float), cudaMemcpyHostToDevice));
  if (targets) CK(cudaMemcpy(h->data_tg, targets, n * HW * sizeof(float), cudaMemcpyHostToDevice));
  else if (h->data_tg) CK(cudaMemcpy(h->data_tg, inputs, n * HW * sizeof(float), cudaMemcpyHostToDevice));
  h->n_data = n;
  return 0;
}

int b2g_autoencoder_train_epoch(b2g_autoencoder* h, const int32_t* order, int64_t n_order, int batch, float lr, double* mean_loss) {
  if (!h || !order || !mean_loss || n_order < 1) return b2g_fail(B2G_EINVAL, "null argument or empty order");
  if (batch < 1 || batch > h->cfg.max_batch) return b2g_fail(B2G_EINVAL, "batch outside [1, max_batch]");
  if (!h->data) return b2g_fail(B2G_ESTATE, "no dataset (b2g_autoencoder_set_dataset first)");
  if (n_order > h->n_data) return b2g_fail(B2G_EINVAL, "order longer than the dataset");
  for (int64_t i = 0; i < n_order; ++i)
    if (order[i] < 0 || order[i] >= h->n_data) return b2g_fail(B2G_EINVAL, "order index outside the dataset");
  if (int rc = need_weights(h)) return rc;
  CK(cudaSetDevice(h->cfg.device));
  if (int rc = upload_lr(h->d_lr, &h->cur_lr, lr, h->stream)) return rc;
  const int rem = (int)(n_order % batch);
  for (int n : {batch, rem}) {
    if (n == 0) continue;
    AePlan* p;
    if (int rc = get_plan(h, n, &p)) return rc;
    if (!p->train)
      if (int rc = capture_graph(h->stream, [&]() { return issue_step(h, *p, n, true, true); }, &p->train)) return rc;
  }
  CK(cudaMemcpyAsync(h->order, order, n_order * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemsetAsync(h->counters + 1, 0, sizeof(long long), h->stream));
  CK(cudaMemsetAsync(h->sumsq, 0, sizeof(double), h->stream));
  for (int64_t s = 0; s + batch <= n_order; s += batch) CK(cudaGraphLaunch(h->plans[batch].train, h->stream));
  if (rem) CK(cudaGraphLaunch(h->plans[rem].train, h->stream));
  double sq = 0;
  CK(cudaMemcpyAsync(&sq, h->sumsq, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  *mean_loss = sq / ((double)n_order * h->cfg.height * h->cfg.width);
  return 0;
}

int b2g_autoencoder_evaluate(b2g_autoencoder* h, int64_t start, int64_t count, double* mean_loss) {
  if (!h || !mean_loss || start < 0 || count < 1) return b2g_fail(B2G_EINVAL, "bad argument");
  if (!h->data || start + count > h->n_data) return b2g_fail(B2G_EINVAL, "slice outside the dataset");
  if (int rc = need_weights(h)) return rc;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemsetAsync(h->sumsq, 0, sizeof(double), h->stream));
  for (int64_t s = 0; s < count; s += h->cfg.max_batch) {
    const int n = (int)std::min<int64_t>(h->cfg.max_batch, count - s);
    AePlan* p;
    if (int rc = get_plan(h, n, &p)) return rc;
    issue_gather(h, n, h->data, h->data_tg ? h->data_tg : h->data, nullptr, nullptr, start + s);
    issue_forward(h, *p, n, false, nullptr);
  }
  CK(cudaGetLastError());
  double sq = 0;
  CK(cudaMemcpyAsync(&sq, h->sumsq, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  *mean_loss = sq / ((double)count * h->cfg.height * h->cfg.width);
  return 0;
}

int b2g_autoencoder_predict(b2g_autoencoder* h, const float* imgs, int n, float* out) {
  if (!h || !imgs || !out || n < 1) return b2g_fail(B2G_EINVAL, "bad argument");
  if (int rc = need_weights(h)) return rc;
  CK(cudaSetDevice(h->cfg.device));
  const size_t HW = (size_t)h->cfg.height * h->cfg.width;
  for (int s = 0; s < n; s += h->cfg.max_batch) {
    const int m = std::min(h->cfg.max_batch, n - s);
    AePlan* p;
    if (int rc = get_plan(h, m, &p)) return rc;
    if (int rc = stage_batch(h, imgs + s * HW, nullptr, m)) return rc;
    issue_forward(h, *p, m, false, h->Y);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(h->pin, h->Y, m * HW * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    memcpy(out + s * HW, h->pin, m * HW * sizeof(float));
  }
  return 0;
}

int b2g_debug_autoencoder_tensor(b2g_autoencoder* h, int layer, int which, float* out, int64_t numel, int32_t* on_tc) {
  if (!h) return b2g_fail(B2G_EINVAL, "null handle");
  if (layer < 0 || layer >= (int)h->L.size()) return b2g_fail(B2G_EINVAL, "layer out of range");
  const AeLayer& y = h->L[layer];
  const size_t N = h->cfg.max_batch;
  const float* src = nullptr;
  size_t n = 0;
  const bool conv = y.kind == ENC_CONV || y.kind == DEC_CONV || y.kind == OUT_CONV;
  switch (which) {
    case 0: src = y.in; n = conv ? N * y.g.hp * y.g.wp * y.g.in_c : N * y.in_ld; break;
    case 1:
      src = y.act;
      n = y.kind == DEC_CONV ? N * y.g.out_h * y.g.out_w * y.g.f : y.kind == ENC_DENSE ? N * h->zs : y.kind == DEC_DENSE ? N * y.g.f : 0;
      break;
    case 2: src = y.D; n = conv ? N * y.dh * y.dw * y.g.f : N * y.dw; break;
    default: return b2g_fail(B2G_EINVAL, "which must be 0 (input), 1 (activation) or 2 (pre-activation gradient)");
  }
  if (!src || n == 0) return b2g_fail(B2G_EINVAL, "layer " + std::to_string(layer) + " keeps no tensor " + std::to_string(which));
  if (on_tc) {   // which engine runs the layer's forward, input gradient and weight gradient (-1: none)
    on_tc[0] = on_tc[1] = on_tc[2] = -1;
    for (const AeGemm& e : h->fwd_g) if (e.d.A == y.in && e.d.B == h->P + y.w_off) on_tc[0] = e.tc;
    for (const AeGemm& e : h->bwd_g) {
      if (e.d.A == y.D && e.d.B == h->P + y.w_off) on_tc[1] = e.tc;
      if (e.wgrad && e.d.A == y.in && e.d.B == y.D) on_tc[2] = e.tc;
    }
  }
  if (!out) return 0;
  if (numel != (int64_t)n) return b2g_fail(B2G_EINVAL, "numel " + std::to_string(numel) + " != " + std::to_string(n));
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaMemcpy(out, src, n * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

int64_t b2g_debug_autoencoder_tensor_numel(b2g_autoencoder* h, int layer, int which) {
  if (!h || layer < 0 || layer >= (int)h->L.size()) return -1;
  const AeLayer& y = h->L[layer];
  const size_t N = h->cfg.max_batch;
  const bool conv = y.kind == ENC_CONV || y.kind == DEC_CONV || y.kind == OUT_CONV;
  if (which == 0) return (int64_t)(conv ? N * y.g.hp * y.g.wp * y.g.in_c : N * y.in_ld);
  if (which == 1)
    return (int64_t)(y.kind == DEC_CONV ? N * y.g.out_h * y.g.out_w * y.g.f : y.kind == ENC_DENSE ? N * h->zs
                                                                              : y.kind == DEC_DENSE ? N * y.g.f : 0);
  if (which == 2) return (int64_t)(conv ? N * y.dh * y.dw * y.g.f : N * y.dw);
  return -1;
}

int b2g_autoencoder_step(b2g_autoencoder* h, const float* inputs, const float* targets, int n, float lr, int apply_update,
                         double* loss) {
  if (!h || !inputs) return b2g_fail(B2G_EINVAL, "null argument");
  if (n < 1 || n > h->cfg.max_batch) return b2g_fail(B2G_EINVAL, "batch " + std::to_string(n) + " outside [1, max_batch]");
  if (int rc = need_weights(h)) return rc;
  CK(cudaSetDevice(h->cfg.device));
  if (int rc = upload_lr(h->d_lr, &h->cur_lr, lr, h->stream)) return rc;
  AePlan* p;
  if (int rc = get_plan(h, n, &p)) return rc;
  CK(cudaMemsetAsync(h->sumsq, 0, sizeof(double), h->stream));
  if (int rc = stage_batch(h, inputs, targets, n)) return rc;
  if (int rc = issue_step(h, *p, n, false, apply_update != 0)) return rc;
  double sq = 0;
  CK(cudaMemcpyAsync(&sq, h->sumsq, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (loss) *loss = sq / ((double)n * h->cfg.height * h->cfg.width);
  return 0;
}

}  // extern "C"
