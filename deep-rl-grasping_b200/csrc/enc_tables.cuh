// Geometry and forward offset tables of the encoder's conv / dense layers, shared by the encoder handle (encoder.cu) and the
// auto-encoder training handle (autoencoder.cu).
//
// TensorFlow 'same' padding (pad_total = max((ceil(in/s)-1)*s + k - in, 0), floor(pad_total/2) in front) is realised by
// keeping each layer's input in a zero-bordered NHWC buffer, so the im2col offset tables need no bounds tests.  Kernels keep
// Keras' HWIO layout, stored with a filter stride rounded up to 4.
#pragma once
#include <algorithm>
#include <string>
#include <vector>

#include "common.cuh"
#include "host.cuh"

namespace b2g {

struct EncLayer {
  int in_h, in_w, in_c;        // logical input
  int k, s, f;                 // kernel, stride, filters (dense: k = s = 0, f = encoding_dim)
  int pad_t, pad_l, hp, wp;    // bordered input geometry
  int out_h, out_w;
  int fs;                      // filter stride of the stored kernel (f rounded up to 4)
  float* in = nullptr;         // bordered input  [N, hp, wp, in_c]
  float* w = nullptr;          // [R, fs]
  float* b = nullptr;          // [fs]
  bool loaded = false;
  int R() const { return k ? k * k * in_c : in_h * in_w * in_c; }
};

// A 'same'-padded conv layer on an [ih, iw, ic] input.
inline EncLayer enc_conv_layer(int ih, int iw, int ic, int k, int s, int f) {
  EncLayer y{};
  y.in_h = ih; y.in_w = iw; y.in_c = ic; y.k = k; y.s = s; y.f = f;
  y.out_h = (ih + s - 1) / s; y.out_w = (iw + s - 1) / s;
  const int ph = std::max((y.out_h - 1) * s + k - ih, 0), pw = std::max((y.out_w - 1) * s + k - iw, 0);
  y.pad_t = ph / 2; y.pad_l = pw / 2; y.hp = ih + ph; y.wp = iw + pw;
  y.fs = (f + 3) / 4 * 4;
  return y;
}

// The encoder's layers for cfg: the convs, then the dense layer.  0, or B2G_EINVAL with the reason set.
inline int enc_geometry(const b2g_encoder_cfg& cfg, std::vector<EncLayer>& layers) {
  int ih = cfg.height, iw = cfg.width, ic = cfg.channels;
  for (int l = 0; l < cfg.n_layers; ++l) {
    if (cfg.kernel[l] < 1 || cfg.strides[l] < 1 || cfg.filters[l] < 1) return b2g_fail(B2G_EINVAL, "bad conv layer spec");
    EncLayer y = enc_conv_layer(ih, iw, ic, cfg.kernel[l], cfg.strides[l], cfg.filters[l]);
    if (l > 0 && (ic & 3)) return b2g_fail(B2G_EINVAL, "hidden conv layers need filters % 4 == 0");
    layers.push_back(y);
    ih = y.out_h; iw = y.out_w; ic = y.f;
  }
  EncLayer dn{};
  dn.in_h = ih; dn.in_w = iw; dn.in_c = ic; dn.k = dn.s = 0; dn.f = cfg.encoding_dim; dn.out_h = dn.out_w = 1;
  dn.hp = ih; dn.wp = iw; dn.fs = (dn.f + 3) / 4 * 4;
  if ((ih * iw * ic) & 3) return b2g_fail(B2G_EINVAL, "flattened feature size must be a multiple of 4");
  layers.push_back(dn);
  return 0;
}

// Offset tables of layer y's forward gather-GEMM over N samples (M = N * out_h * out_w rows, R = y.R()).  The output lands at
// row (b, oy, ox) of an [o_hp, o_wp, o_c] map with the interior starting at (o_pt, o_pl); a dense layer's input rows are R wide.
inline void enc_fwd_tables(const EncLayer& y, int N, int o_hp, int o_wp, int o_pt, int o_pl, int o_c, std::vector<int>& aM,
                           std::vector<int>& cM, std::vector<int>& aR, std::vector<int>& bR, std::vector<int>& bN,
                           std::vector<int>& cN) {
  const bool dense = y.k == 0;
  const int M = N * y.out_h * y.out_w, R = y.R();
  aM.assign(M, 0); cM.assign(M, 0); aR.assign(R, 0); bR.assign(R, 0); bN.assign(y.f, 0); cN.assign(y.f, 0);
  for (int b = 0; b < N; ++b)
    for (int oy = 0; oy < y.out_h; ++oy)
      for (int ox = 0; ox < y.out_w; ++ox) {
        const int m = (b * y.out_h + oy) * y.out_w + ox;
        aM[m] = dense ? b * R : ((b * y.hp + oy * y.s) * y.wp + ox * y.s) * y.in_c;
        cM[m] = ((b * o_hp + oy + o_pt) * o_wp + ox + o_pl) * o_c;
      }
  for (int r = 0; r < R; ++r) {
    if (dense) aR[r] = r;
    else {
      const int c = r % y.in_c, kx = (r / y.in_c) % y.k, ky = r / (y.in_c * y.k);
      aR[r] = (ky * y.wp + kx) * y.in_c + c;
    }
    bR[r] = r * y.fs;
  }
  for (int n = 0; n < y.f; ++n) bN[n] = cN[n] = n;
}

// Engine flags of that forward: bias + LeakyReLU epilogue; element-wise A gathers when the input channels break 4-groups.
inline int enc_fwd_flags(const EncLayer& y) {
  return GG_A_RVEC | GG_EPI_BIAS_LRELU | ((y.in_c & 3) && y.k ? GG_A_SCALAR : 0);
}

}  // namespace b2g
