// libb200grasp: SAC learner handle, HBM layout, offset tables, step orchestration, C ABI.
//
// HBM layout (all fp32 unless noted; everything is allocated once in b2g_sac_create, except the opt-in obs_rms and observe
// staging of obsnorm.cu, allocated by b2g_obs_rms_set and the first b2g_sac_observe_* call):
//   P  : parameter arena  [ model/pi | model/values_fn | log_ent_coef | target/values_fn ], every
//        tensor padded to 32 floats, tensor order = SB zip parameter_list (SURVEY.md Appendix B)
//   Mo, Vo, G : Adam moments and gradients, same offsets as the trainable part of P
//   replay  : frames[frame_cap][frame_bytes] (raw, un-normalised compact rows, RGB planes optionally uint8; replay.cu)
//             obs_frame[cap] next_frame[cap] (int32) act[cap,A] rew[cap] done[cap]
//   batch   : x_obs/x_next [B,H,W,C] (normalised, /255), h1/h2/h3 per network, F rows [B,FS]
//             (512 CNN features | direct feature | replay action | zero pad), gradient maps with
//             zero borders (dZ3p, dZ2p) so the dgrad gathers need no bounds logic
// One gradient step = prep -> gather -> zero G -> forward contractions -> tail -> backward contractions
// -> [all-reduce of G] -> optim; captured once in a CUDA graph and replayed.  The 64x64 CNN policy in
// bf16x3 runs its contractions on engine v2 (engine_v2.cu: one fused forward and one fused backward
// launch); every other configuration, and policy inference, runs them as grouped launches of the
// round-1 engines (gg_tc.cu, gg_simt.cu).
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <map>
#include <tuple>
#include <string>
#include <vector>

#include "../../include/b200grasp.h"
#include "common.cuh"
#include "sac_internal.cuh"
#include "state.cuh"

using namespace b2g;

namespace b2g {
bool pdl_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("B2G_PDL"); v = (e && e[0] == '0') ? 0 : 1; }
  return v != 0;
}
}  // namespace b2g

namespace {

int64_t pad32(int64_t n) { return (n + 31) / 32 * 32; }

// layer scopes conv1, conv2, conv3, fc1 of each extractor (b2g_sac_net_cfg): create_augmented_nature_cnn's, and stable-baselines'
// nature_cnn (common/policies.py: conv(.., 'c1'), 'c2', 'c3', linear(.., 'fc1'))
const char* const kCnnScopes[2][4] = {{"cnn1", "cnn2", "cnn3", "cnn_fc1"}, {"c1", "c2", "c3", "fc1"}};

void add_tensor(b2g_sac* h, const std::string& name, std::vector<int64_t> shape, int group) {
  Tensor t;
  t.name = name;
  t.ndim = (int)shape.size();
  t.numel = 1;
  for (int i = 0; i < 4; ++i) t.shape[i] = i < t.ndim ? shape[i] : 1;
  for (auto s : shape) t.numel *= s;
  t.group = group;
  t.off = 0;
  h->tindex[name] = (int)h->tensors.size();
  h->tensors.push_back(t);
}

void add_cnn(b2g_sac* h, const std::string& pre, int group) {
  add_tensor(h, h->cnn_t(pre, 0, "w"), {8, 8, h->Cimg, 32}, group);
  add_tensor(h, h->cnn_t(pre, 0, "b"), {1, 32, 1, 1}, group);
  add_tensor(h, h->cnn_t(pre, 1, "w"), {4, 4, 32, 64}, group);
  add_tensor(h, h->cnn_t(pre, 1, "b"), {1, 64, 1, 1}, group);
  add_tensor(h, h->cnn_t(pre, 2, "w"), {3, 3, 64, 64}, group);
  add_tensor(h, h->cnn_t(pre, 2, "b"), {1, 64, 1, 1}, group);
  add_tensor(h, h->cnn_t(pre, 3, "w"), {1024, 512}, group);
  add_tensor(h, h->cnn_t(pre, 3, "b"), {512}, group);
}
void add_mlp(b2g_sac* h, const std::string& pre, int in_dim, int group) {
  add_tensor(h, pre + "/fc0/kernel", {in_dim, h->H}, group);
  add_tensor(h, pre + "/fc0/bias", {h->H}, group);
  add_tensor(h, h->fc1(pre) + "/kernel", {h->H, h->H}, group);
  add_tensor(h, h->fc1(pre) + "/bias", {h->H}, group);
}

// Parameter inventory in SB-zip order (oracle/sac_ref.py param_specs; SURVEY.md Appendix B)
void build_params(b2g_sac* h) {
  const int A = h->A, H = h->H, fd = h->feat_dim;
  if (h->cnn) add_cnn(h, "model/pi", 0);
  add_mlp(h, "model/pi", fd, 0);
  add_tensor(h, "model/pi/dense/kernel", {H, A}, 0);
  add_tensor(h, "model/pi/dense/bias", {A}, 0);
  add_tensor(h, "model/pi/dense_1/kernel", {H, A}, 0);
  add_tensor(h, "model/pi/dense_1/bias", {A}, 0);
  for (int tgt = 0; tgt < 2; ++tgt) {
    const std::string sc = tgt ? "target/values_fn" : "model/values_fn";
    const int grp = tgt ? 3 : 1;
    if (h->cnn) add_cnn(h, sc, grp);
    add_mlp(h, sc + "/vf", fd, grp);
    add_tensor(h, sc + "/vf/vf/kernel", {H, 1}, grp);
    add_tensor(h, sc + "/vf/vf/bias", {1}, grp);
    if (!tgt) {
      for (const char* q : {"qf1", "qf2"}) {
        add_mlp(h, sc + "/" + q, fd + A, grp);
        add_tensor(h, sc + "/" + q + "/" + q + "/kernel", {H, 1}, grp);
        add_tensor(h, sc + "/" + q + "/" + q + "/bias", {1}, grp);
      }
      add_tensor(h, "model/log_ent_coef", {}, 2);
    }
  }
  int64_t off = 0;
  int64_t gstart[5] = {0, 0, 0, 0, 0};
  int cur = 0;
  for (auto& t : h->tensors) {
    while (cur < t.group) gstart[++cur] = off;
    t.off = off;
    off += pad32(t.numel);
  }
  while (cur < 4) gstart[++cur] = off;
  h->n_pi = gstart[1] - gstart[0];
  h->n_values = gstart[2] - gstart[1];
  h->n_ent = gstart[3] - gstart[2];
  h->n_target = gstart[4] - gstart[3];
  h->n_train = gstart[3];
  h->n_all = off;
}

// SAC's passes over a group before the shared tile layout: GG_CN_AFFINE4 and column-table ids (gg_tc_columns), split-R, flops
int finalize_group(b2g_sac* h, GemmGroup& g) {
  g.flops = 0;
  const int bm = g.tc ? GG_TC_BM : GG_SIMT_BM, bn = g.tc ? GG_TC_BN : GG_SIMT_BN, bk = g.tc ? GG_TC_BK : GG_SIMT_BK;
  for (auto& d : g.host) {
    gg_tc_columns(d, h->host_tabs, h->col_ids);
    if (d.flags & GG_EPI_ATOMIC) {     // split-R sized for this engine's tile grid
      const int tiles = ((d.M + bm - 1) / bm) * ((d.N + bn - 1) / bn);
      int sp = std::max(1, h->num_sms / std::max(1, tiles));
      sp = std::min(sp, std::max(1, d.R / (2 * bk)));
      d.splitR = sp;
    }
    g.flops += 2.0 * d.M * d.N * d.R;
  }
  return finalize_tiles(g, h->allocs, h->stream, bm, bn);
}

int split_for(int tiles, int R, int target_ctas = 132) {
  int s = std::max(1, target_ctas / std::max(1, tiles));
  const int max_s = std::max(1, R / (4 * GG_SIMT_BK));
  return std::min(s, max_s);
}

#define TAB(var, vec)                                         \
  const int* var = nullptr;                                   \
  if (int rc_ = upload_table(h->allocs, h->stream, (vec), &var, &h->host_tabs)) return rc_;

int build_groups(b2g_sac* h) {
  const int B = h->B, A = h->A, H = h->H, FS = h->FS, fd = h->feat_dim;
  const char* nets[3] = {"model/pi", "model/values_fn", "target/values_fn"};
  TAB(i64, iota_tab(64));           // generic small iotas
  TAB(i512, iota_tab(512));
  TAB(i1024, iota_tab(1024));
  TAB(rowH, iota_tab(B, H));        // b*H
  TAB(rowFS, iota_tab(B, FS));
  TAB(row3H, iota_tab(B, 3 * H));
  TAB(iFS, iota_tab(FS));
  TAB(iH, iota_tab(H));             // head columns
  TAB(kH, iota_tab(std::max(FS, H), H));   // j*H  (fc0 / fc1 kernel rows)

  auto nn = [&](int net, const char* s) { return std::string(nets[net]) + s; };
  auto ct = [&](int net, int layer, const char* wb) { return h->cnn_t(nets[net], layer, wb); };

  if (h->cnn) {
    const int Ci = h->Cimg, Hi = h->Hi, Wi = h->Wi, H1 = h->H1, W1 = h->W1, H2 = h->H2, W2 = h->W2, H3 = h->H3, W3 = h->W3;
    const int P2h = H2 + 3, P2w = W2 + 3, P3h = H3 + 4, P3w = W3 + 4;
    // ---- forward / wgrad tables per conv layer
    struct Conv { int Hi, Wi, Ci, k, s, Ho, Wo, Co; };
    const Conv cv[3] = {{Hi, Wi, Ci, 8, 4, H1, W1, 32}, {H1, W1, 32, 4, 2, H2, W2, 64}, {H2, W2, 64, 3, 1, H3, W3, 64}};
    const int* rowoff[3]; const int* koff[3]; const int* wrow[3]; const int* crow[3];
    for (int l = 0; l < 3; ++l) {
      const Conv& c = cv[l];
      std::vector<int> ro(B * c.Ho * c.Wo), ko(c.k * c.k * c.Ci);
      for (int b = 0; b < B; ++b)
        for (int oy = 0; oy < c.Ho; ++oy)
          for (int ox = 0; ox < c.Wo; ++ox)
            ro[(b * c.Ho + oy) * c.Wo + ox] = ((b * c.Hi + oy * c.s) * c.Wi + ox * c.s) * c.Ci;
      for (int ky = 0; ky < c.k; ++ky)
        for (int kx = 0; kx < c.k; ++kx)
          for (int ci = 0; ci < c.Ci; ++ci) ko[(ky * c.k + kx) * c.Ci + ci] = (ky * c.Wi + kx) * c.Ci + ci;
      if (int rc = upload_table(h->allocs, h->stream, ro, &rowoff[l], &h->host_tabs)) return rc;
      if (int rc = upload_table(h->allocs, h->stream, ko, &koff[l], &h->host_tabs)) return rc;
      if (int rc = upload_table(h->allocs, h->stream, iota_tab(c.k * c.k * c.Ci, c.Co), &wrow[l], &h->host_tabs)) return rc;
      if (int rc = upload_table(h->allocs, h->stream, iota_tab(B * c.Ho * c.Wo, c.Co), &crow[l], &h->host_tabs)) return rc;
    }
    TAB(fcA, iota_tab(B, 1024));
    TAB(fcW, iota_tab(1024, 512));
    // transposed weight planes [N][R]: element (r, n) at n*R + r
    const int* wT_r[4]; const int* wT_n[4];
    {
      const int Rs[4] = {64 * Ci, 512, 576, 1024}, Ns[4] = {32, 64, 64, 512};
      for (int l = 0; l < 4; ++l) {
        if (int rc = upload_table(h->allocs, h->stream, iota_tab(Rs[l]), &wT_r[l], &h->host_tabs)) return rc;
        if (int rc = upload_table(h->allocs, h->stream, iota_tab(Ns[l], Rs[l]), &wT_n[l], &h->host_tabs)) return rc;
      }
    }
    // ================= forward groups
    for (int l = 0; l < 3; ++l) {
      const Conv& c = cv[l];
      GemmGroup g;
      g.name = std::string("conv") + char('1' + l) + "_fwd";
      for (int n = 0; n < 3; ++n) {
        const float* in = l == 0 ? (n == 2 ? h->x_next : h->x_obs) : (l == 1 ? h->h1[n] : h->h2[n]);
        float* out = l == 0 ? h->h1[n] : (l == 1 ? h->h2[n] : h->h3[n]);
        GemmDesc d = gemm_desc(in, rowoff[l], koff[l], h->p(ct(n, l, "w")), wrow[l], i64, out, crow[l], i64,
                        B * c.Ho * c.Wo, c.Co, c.k * c.k * c.Ci, GG_A_RVEC | GG_EPI_BIAS_RELU);
        d.bias = h->p(ct(n, l, "b"));
        if (h->use_planes) {
          uint16_t* const* ip = l == 0 ? h->xp[n == 2 ? 1 : 0] : (l == 1 ? h->h1p[n] : h->h2p[n]);
          uint16_t* const* op = l == 0 ? h->h1p[n] : (l == 1 ? h->h2p[n] : h->h3p[n]);
          d.flags |= GG_PLANES | GG_B_RVEC | ((l == 0 && (c.Ci & 1)) ? GG_A_ALIGN4 : 0) | (l == 0 ? GG_A_ROWLANES : 0);
          d.A_hi = ip[0]; d.A_lo = ip[1];
          d.B_hi = h->wp[n][l][2]; d.B_lo = h->wp[n][l][3];
          d.bR_p = wT_r[l]; d.bN_p = wT_n[l];
          d.C_hi = op[0]; d.C_lo = op[1];
        }
        g.host.push_back(d);
      }
      h->fwd_groups.push_back(g);
    }
    {
      GemmGroup g;
      g.name = "fc1_fwd";
      for (int n = 0; n < 3; ++n) {
        GemmDesc d = gemm_desc(h->h3[n], fcA, i1024, h->p(ct(n, 3, "w")), fcW, i512, h->F[n], rowFS, i512, B, 512, 1024,
                        GG_A_RVEC | GG_EPI_BIAS_RELU);
        d.bias = h->p(ct(n, 3, "b"));
        if (h->use_planes) {
          d.flags |= GG_PLANES | GG_B_RVEC;
          d.A_hi = h->h3p[n][0]; d.A_lo = h->h3p[n][1];
          d.B_hi = h->wp[n][3][2]; d.B_lo = h->wp[n][3][3];
          d.bR_p = wT_r[3]; d.bN_p = wT_n[3];
        }
        g.host.push_back(d);
      }
      h->fwd_groups.push_back(g);
    }
    // policy-inference groups (pi network only)
    for (int l = 0; l < 4; ++l) {
      GemmGroup g = h->fwd_groups[l];
      g.name = "act_" + g.name;
      g.host.resize(1);
      g.dev = nullptr;
      h->act_groups.push_back(g);
    }

    if (!h->v2.on) {     // the round-1 backward: built only when the round-1 engines train
      // dZ row tables in the zero-bordered layouts
      std::vector<int> z2row(B * H2 * W2), z3row(B * H3 * W3);
      for (int b = 0; b < B; ++b) {
        for (int y = 0; y < H2; ++y)
          for (int x = 0; x < W2; ++x) z2row[(b * H2 + y) * W2 + x] = ((b * P2h + y + 1) * P2w + x + 1) * 64;
        for (int y = 0; y < H3; ++y)
          for (int x = 0; x < W3; ++x) z3row[(b * H3 + y) * W3 + x] = ((b * P3h + y + 2) * P3w + x + 2) * 64;
      }
      TAB(dz2row, z2row);
      TAB(dz3row, z3row);
      // ================= backward groups (pi, values)
      // head dgrad -> dZ4 (masked by relu of cnn_fc1 output)
      {
        GemmGroup g;
        g.name = "heads_dgrad";
        TAB(row512, iota_tab(B, 512));
        // pi
        GemmDesc d = gemm_desc(h->dz0_pi, rowH, iH, h->p("model/pi/fc0/kernel"), iH, kH, h->dZ4[0], row512, i512, B, 512, H,
                        GG_A_RVEC | GG_B_RVEC | GG_EPI_MASK);
        d.mask = h->F[0]; d.kM = rowFS; d.kN = i512;
        if (h->use_planes) { d.C_hi = h->dZ4p[0][0]; d.C_lo = h->dZ4p[0][1]; }
        g.host.push_back(d);
        // values: [dz0_vf | dz0_q1 | dz0_q2] x [K0_vf ; K0_q1 ; K0_q2]^T
        std::vector<int> br(3 * H);
        const char* hn[3] = {"/vf/fc0/kernel", "/qf1/fc0/kernel", "/qf2/fc0/kernel"};
        for (int q = 0; q < 3; ++q)
          for (int r = 0; r < H; ++r) br[q * H + r] = (int)(h->tensors[h->tindex.at(nn(1, hn[q]))].off) + r;
        TAB(brv, br);
        TAB(i3H, iota_tab(3 * H));
        GemmDesc e = gemm_desc(h->dz0_v3, row3H, i3H, h->P, brv, kH, h->dZ4[1], row512, i512, B, 512, 3 * H,
                        GG_A_RVEC | GG_B_RVEC | GG_EPI_MASK);
        e.mask = h->F[1]; e.kM = rowFS; e.kN = i512;
        if (h->use_planes) { e.C_hi = h->dZ4p[1][0]; e.C_lo = h->dZ4p[1][1]; }
        g.host.push_back(e);
        h->bwd_groups.push_back(g);
        // fc1 wgrad + dgrad
        GemmGroup f;
        f.name = "fc1_bwd";
        std::vector<int> cn(1024), fcT(1024);
        for (int y = 0; y < H3; ++y)
          for (int x = 0; x < W3; ++x)
            for (int c = 0; c < 64; ++c) cn[(y * W3 + x) * 64 + c] = ((y + 2) * P3w + (x + 2)) * 64 + c;
        TAB(cN3p, cn);
        TAB(rowP3, iota_tab(B, P3h * P3w * 64));
        TAB(wfT, iota_tab(1024, 512));
        for (int n = 0; n < 2; ++n) {
          GemmDesc w = gemm_desc(h->h3[n], i1024, fcA, h->dZ4[n], row512, i512, h->g(ct(n, 3, "w")), fcW, i512, 1024, 512, B,
                          GG_COLSUM);
          w.colsum = h->g(ct(n, 3, "b"));
          if (h->use_planes) {
            w.flags = (w.flags & ~GG_COLSUM) | GG_PLANES | GG_MN_MAJOR;
            w.A_hi = h->h3p[n][0]; w.A_lo = h->h3p[n][1]; w.B_hi = h->dZ4p[n][0]; w.B_lo = h->dZ4p[n][1];
          }
          f.host.push_back(w);
          GemmDesc dg = gemm_desc(h->dZ4[n], row512, i512, h->p(ct(n, 3, "w")), i512, wfT, h->dZ3p[n], rowP3, cN3p, B, 1024, 512,
                           GG_A_RVEC | GG_B_RVEC | GG_EPI_MASK);
          dg.mask = h->h3[n]; dg.kM = fcA; dg.kN = i1024;
          if (h->use_planes) {
            dg.flags |= GG_PLANES;
            dg.A_hi = h->dZ4p[n][0]; dg.A_lo = h->dZ4p[n][1];
            dg.B_hi = h->wp[n][3][0]; dg.B_lo = h->wp[n][3][1];
            dg.C_hi = h->dZ3pp[n][0]; dg.C_lo = h->dZ3pp[n][1];
          }
          f.host.push_back(dg);
        }
        h->bwd_groups.push_back(f);
      }
      // conv3 wgrad + dgrad
      {
        GemmGroup g;
        g.name = "conv3_bwd";
        std::vector<int> am(B * H2 * W2), ar(9 * 64), br(9 * 64), cm(B * H2 * W2);
        for (int b = 0; b < B; ++b)
          for (int y = 0; y < H2; ++y)
            for (int x = 0; x < W2; ++x) {
              am[(b * H2 + y) * W2 + x] = ((b * P3h + y + 2) * P3w + x + 2) * 64;
              cm[(b * H2 + y) * W2 + x] = ((b * P2h + y + 1) * P2w + x + 1) * 64;
            }
        for (int ky = 0; ky < 3; ++ky)
          for (int kx = 0; kx < 3; ++kx)
            for (int n = 0; n < 64; ++n) {
              ar[(ky * 3 + kx) * 64 + n] = -(ky * P3w + kx) * 64 + n;
              br[(ky * 3 + kx) * 64 + n] = (ky * 3 + kx) * 64 * 64 + n;
            }
        TAB(t_am, am); TAB(t_ar, ar); TAB(t_br, br); TAB(t_cm, cm);
        TAB(c64, iota_tab(64, 64));
        const int R = B * H3 * W3;
        for (int n = 0; n < 2; ++n) {
          GemmDesc w = gemm_desc(h->h2[n], koff[2], rowoff[2], h->dZ3p[n], dz3row, i64, h->g(ct(n, 2, "w")), wrow[2], i64, 576, 64, R,
                          GG_COLSUM | GG_EPI_ATOMIC, split_for(9, R));
          w.colsum = h->g(ct(n, 2, "b"));
          if (h->use_planes) {
            w.flags = (w.flags & ~GG_COLSUM) | GG_PLANES | GG_MN_MAJOR;
            w.A_hi = h->h2p[n][0]; w.A_lo = h->h2p[n][1]; w.B_hi = h->dZ3pp[n][0]; w.B_lo = h->dZ3pp[n][1];
          }
          g.host.push_back(w);
          GemmDesc dg = gemm_desc(h->dZ3p[n], t_am, t_ar, h->p(ct(n, 2, "w")), t_br, c64, h->dZ2p[n], t_cm, i64, B * H2 * W2, 64, 576,
                           GG_A_RVEC | GG_B_RVEC | GG_EPI_MASK);
          dg.mask = h->h2[n]; dg.kM = crow[1]; dg.kN = i64;
          if (h->use_planes) {
            dg.flags |= GG_PLANES;
            dg.A_hi = h->dZ3pp[n][0]; dg.A_lo = h->dZ3pp[n][1];
            dg.B_hi = h->wp[n][2][0]; dg.B_lo = h->wp[n][2][1];
            dg.C_hi = h->dZ2pp[n][0]; dg.C_lo = h->dZ2pp[n][1];
          }
          g.host.push_back(dg);
        }
        h->bwd_groups.push_back(g);
      }
      // conv2 wgrad + 4 parity-class dgrads
      {
        GemmGroup g;
        g.name = "conv2_bwd";
        const int R = B * H2 * W2;
        TAB(c64, iota_tab(32, 64));
        for (int n = 0; n < 2; ++n) {
          GemmDesc w = gemm_desc(h->h1[n], koff[1], rowoff[1], h->dZ2p[n], dz2row, i64, h->g(ct(n, 1, "w")), wrow[1], i64, 512, 64, R,
                          GG_COLSUM | GG_EPI_ATOMIC, split_for(8, R));
          w.colsum = h->g(ct(n, 1, "b"));
          if (h->use_planes) {
            w.flags = (w.flags & ~GG_COLSUM) | GG_PLANES | GG_MN_MAJOR;
            w.A_hi = h->h1p[n][0]; w.A_lo = h->h1p[n][1]; w.B_hi = h->dZ2pp[n][0]; w.B_lo = h->dZ2pp[n][1];
          }
          g.host.push_back(w);
        }
        for (int py = 0; py < 2; ++py)
          for (int px = 0; px < 2; ++px) {
            const int ny = (H1 - py + 1) / 2, nx = (W1 - px + 1) / 2;
            std::vector<int> am(B * ny * nx), cm(B * ny * nx), ar(4 * 64), br(4 * 64);
            for (int b = 0; b < B; ++b)
              for (int yy = 0; yy < ny; ++yy)
                for (int xx = 0; xx < nx; ++xx) {
                  am[(b * ny + yy) * nx + xx] = ((b * P2h + yy + 1) * P2w + xx + 1) * 64;
                  cm[(b * ny + yy) * nx + xx] = ((b * H1 + 2 * yy + py) * W1 + 2 * xx + px) * 32;
                }
            for (int jy = 0; jy < 2; ++jy)
              for (int jx = 0; jx < 2; ++jx)
                for (int q = 0; q < 64; ++q) {
                  ar[(jy * 2 + jx) * 64 + q] = -(jy * P2w + jx) * 64 + q;
                  br[(jy * 2 + jx) * 64 + q] = (((py + 2 * jy) * 4 + (px + 2 * jx)) * 32) * 64 + q;
                }
            TAB(t_am, am); TAB(t_ar, ar); TAB(t_br, br); TAB(t_cm, cm);
            for (int n = 0; n < 2; ++n) {
              GemmDesc dg = gemm_desc(h->dZ2p[n], t_am, t_ar, h->p(ct(n, 1, "w")), t_br, c64, h->dZ1[n], t_cm, i64, B * ny * nx, 32, 256,
                               GG_A_RVEC | GG_B_RVEC | GG_EPI_MASK);
              dg.mask = h->h1[n];
              if (h->use_planes) {
                dg.flags |= GG_PLANES;
                dg.A_hi = h->dZ2pp[n][0]; dg.A_lo = h->dZ2pp[n][1];
                dg.B_hi = h->wp[n][1][0]; dg.B_lo = h->wp[n][1][1];
                dg.C_hi = h->dZ1p[n][0]; dg.C_lo = h->dZ1p[n][1];
              }
              g.host.push_back(dg);
            }
          }
        h->bwd_groups.push_back(g);
      }
      // conv1 wgrad
      {
        GemmGroup g;
        g.name = "conv1_wgrad";
        const int R = B * H1 * W1, M = 64 * Ci;
        for (int n = 0; n < 2; ++n) {
          GemmDesc w = gemm_desc(h->x_obs, koff[0], rowoff[0], h->dZ1[n], crow[0], i64, h->g(ct(n, 0, "w")), wrow[0], i64, M, 32, R,
                          GG_COLSUM | GG_EPI_ATOMIC, split_for((M + 63) / 64, R, 74));
          w.colsum = h->g(ct(n, 0, "b"));
          if (h->use_planes) {
            w.flags = (w.flags & ~GG_COLSUM) | GG_PLANES | GG_MN_MAJOR | ((Ci & 1) ? GG_A_ALIGN4 : 0) | GG_A_ROWLANES;
            w.A_hi = h->xp[0][0]; w.A_lo = h->xp[0][1]; w.B_hi = h->dZ1p[n][0]; w.B_lo = h->dZ1p[n][1];
          }
          g.host.push_back(w);
        }
        h->bwd_groups.push_back(g);
      }
      if (h->use_planes) {     // bias gradients (column sums of the gradient maps) as one small launch
        TAB(row512b, iota_tab(B, 512));
        std::vector<ColsumJob> jobs, early;
        int start = 0, estart = 0;
        for (int n = 0; n < 2; ++n) {
          const float* srcs[4] = {h->dZ1[n], h->dZ2p[n], h->dZ3p[n], h->dZ4[n]};
          const int* rows[4] = {crow[0], dz2row, dz3row, row512b};
          const int nrows[4] = {B * H1 * W1, B * H2 * W2, B * H3 * W3, B};
          const int Ns[4] = {32, 64, 64, 512};
          for (int l = 0; l < 4; ++l) {
            const int rows_per_cta = 8 * (256 / (Ns[l] / 4));
            const int ctas = (nrows[l] + rows_per_cta - 1) / rows_per_cta;
            if (l == 3) {       // cnn_fc1 bias: ready as soon as dZ4 exists -> part of the early all-reduce range
              early.push_back(ColsumJob{srcs[l], rows[l], h->g(ct(n, l, "b")), nrows[l], Ns[l], estart});
              estart += ctas;
            } else {
              jobs.push_back(ColsumJob{srcs[l], rows[l], h->g(ct(n, l, "b")), nrows[l], Ns[l], start});
              start += ctas;
            }
          }
        }
        h->n_colsum_early = (int)early.size();
        h->colsum_early_ctas = estart;
        if (int rc = dev_alloc(h->allocs, h->stream, &h->d_colsum_early, early.size(), false)) return rc;
        CK(cudaMemcpyAsync(h->d_colsum_early, early.data(), early.size() * sizeof(ColsumJob), cudaMemcpyHostToDevice, h->stream));
        h->n_colsum = (int)jobs.size();
        h->colsum_ctas = start;
        if (int rc = dev_alloc(h->allocs, h->stream, &h->d_colsum, jobs.size(), false)) return rc;
        CK(cudaMemcpyAsync(h->d_colsum, jobs.data(), jobs.size() * sizeof(ColsumJob), cudaMemcpyHostToDevice, h->stream));
        CK(cudaStreamSynchronize(h->stream));
      }
    }
  }

  // ================= heads fc0 forward (all policies)
  {
    GemmGroup g;
    g.name = "heads_fc0";
    const char* hk[5] = {"model/pi/fc0/kernel", "model/values_fn/vf/fc0/kernel", "model/values_fn/qf1/fc0/kernel",
                         "model/values_fn/qf2/fc0/kernel", "target/values_fn/vf/fc0/kernel"};
    const int fnet[5] = {0, 1, 1, 1, 2};
    for (int q = 0; q < 5; ++q) {
      const int R = (q == 2 || q == 3) ? fd + A : fd;
      g.host.push_back(gemm_desc(h->F[fnet[q]], rowFS, iFS, h->p(hk[q]), kH, iH, h->z0[q], rowH, iH, B, H, R, GG_A_RVEC));
    }
    GemmGroup a = g;
    // training step: the 516-deep reduction of each head is split over several CTAs (atomic accumulation into the
    // pre-zeroed z0 block) -- 10 tiles would otherwise each walk 9 r-chunks serially on 10 of the 132 SMs
    for (auto& d : g.host) d.flags |= GG_EPI_ATOMIC;
    h->fwd_groups.push_back(g);
    a.name = "act_heads_fc0";
    a.host.resize(1);
    h->act_groups.push_back(a);
  }
  // ================= heads wgrad (fc0 and fc1 kernels + their biases through COLSUM)
  if (!h->v2.on) {     // (engine v2 steps compute them with heads_wgrad_kernel, tail.cu)
    GemmGroup g;
    g.name = "heads_wgrad";
    const char* hp[4] = {"model/pi", "model/values_fn/vf", "model/values_fn/qf1", "model/values_fn/qf2"};
    TAB(i3Hs0, iota_tab(B, 3 * H, 0));
    TAB(i3Hs1, iota_tab(B, 3 * H, H));
    TAB(i3Hs2, iota_tab(B, 3 * H, 2 * H));
    const int* dzrow[4] = {rowH, i3Hs0, i3Hs1, i3Hs2};
    for (int q = 0; q < 4; ++q) {
      const int M = (q >= 2) ? fd + A : fd;
      const float* dz0 = q == 0 ? h->dz0_pi : h->dz0_v3;
      GemmDesc w0 = gemm_desc(h->F[q == 0 ? 0 : 1], iFS, rowFS, dz0, dzrow[q], iH, h->g(std::string(hp[q]) + "/fc0/kernel"), kH, iH, M, H, B,
                       GG_COLSUM);
      w0.colsum = h->g(std::string(hp[q]) + "/fc0/bias");
      g.host.push_back(w0);
      GemmDesc w1 = gemm_desc(h->a0[q], iH, rowH, h->dz1[q], rowH, iH, h->g(h->fc1(hp[q]) + "/kernel"), kH, iH, H, H, B, GG_COLSUM);
      w1.colsum = h->g(h->fc1(hp[q]) + "/bias");
      g.host.push_back(w1);
    }
    // heads_wgrad must run before heads_dgrad? no dependency; keep it first in the backward list
    h->bwd_groups.insert(h->bwd_groups.begin(), g);
  }
  if (h->use_planes) {
    const int Rs[4] = {64 * h->Cimg, 512, 576, 1024}, Ns[4] = {32, 64, 64, 512};
    std::vector<PlaneJob> jobs;
    int start = 0;
    for (int n = 0; n < 3; ++n)
      for (int l = 0; l < 4; ++l) {
        PlaneJob j{};
        j.src = h->p(h->cnn_t(nets[n], l, "w"));
        j.hi = h->wp[n][l][0]; j.lo = h->wp[n][l][1]; j.hiT = h->wp[n][l][2]; j.loT = h->wp[n][l][3];
        j.R = Rs[l]; j.N = Ns[l]; j.tile_start = start;
        start += ((j.R + 31) / 32) * ((j.N + 31) / 32);
        jobs.push_back(j);
      }
    h->n_jobs = (int)jobs.size();
    h->job_tiles = start;
    if (int rc = dev_alloc(h->allocs, h->stream, &h->d_jobs, jobs.size(), false)) return rc;
    CK(cudaMemcpyAsync(h->d_jobs, jobs.data(), jobs.size() * sizeof(PlaneJob), cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  // one operand-contiguity mode per launch (the wgmma kernel is specialised on it): split mixed groups
  {
    std::vector<GemmGroup> split;
    for (auto& g : h->bwd_groups) {
      std::vector<GemmDesc> wg, dg;
      for (auto& d : g.host) ((d.flags & GG_A_RVEC) ? dg : wg).push_back(d);
      // the cp.async (planes) kernel picks K-major / MN-major per tile at run time, so a layer's wgrad and dgrad
      // share one launch when every problem of the group is in planes mode
      bool all_planes = true;
      for (auto& d : g.host) all_planes = all_planes && (d.flags & GG_PLANES);
      if (wg.empty() || dg.empty() || all_planes) { split.push_back(g); continue; }
      GemmGroup a = g, b = g;
      const std::string base = g.name.substr(0, g.name.find('_'));
      a.name = base + "_wgrad"; a.host = wg;
      b.name = base + "_dgrad"; b.host = dg;
      split.push_back(a); split.push_back(b);
    }
    h->bwd_groups.swap(split);
  }
  // engine selection: the large dense contractions (convs, cnn_fc1, head fc0) go to the wgmma engine unless fp32 SIMT is asked for
  auto pick = [&](GemmGroup& g) {
    g.tc = h->cfg.precision != B2G_PREC_FP32_SIMT && (g.name.find("conv") != std::string::npos || g.name.find("fc1_") != std::string::npos ||
                                                        g.name.find("heads_") != std::string::npos);
  };
  // engine v2 runs the training forward: of the round-1 forward groups only their policy-inference copies are launched
  if (h->v2.on) h->fwd_groups.clear();
  for (auto& g : h->fwd_groups) { pick(g); if (int rc = finalize_group(h, g)) return rc; }
  for (auto& g : h->bwd_groups) { pick(g); if (int rc = finalize_group(h, g)) return rc; }
  for (auto& g : h->act_groups) { pick(g); if (int rc = finalize_group(h, g)) return rc; }
  return 0;
}

HeadW head_w(b2g_sac* h, const std::string& pre, const std::string& out) {
  HeadW w;
  w.k0 = h->p(pre + "/fc0/kernel");
  w.b0 = h->p(pre + "/fc0/bias");
  w.k1 = h->p(h->fc1(pre) + "/kernel");
  w.b1 = h->p(h->fc1(pre) + "/bias");
  w.ko = h->p(pre + "/" + out + "/kernel");
  w.bo = h->p(pre + "/" + out + "/bias");
  return w;
}
HeadG head_g(b2g_sac* h, const std::string& pre, const std::string& out) {
  HeadG g;
  g.b1 = h->g(h->fc1(pre) + "/bias");
  g.ko = h->g(pre + "/" + out + "/kernel");
  g.bo = h->g(pre + "/" + out + "/bias");
  return g;
}

TailArgs make_tail(b2g_sac* h, bool want_per_sample) {
  TailArgs t{};
  t.B = h->B; t.H = h->H; t.A = h->A; t.feat_dim = h->feat_dim;
  t.gamma = h->cfg.gamma; t.target_entropy = h->cfg.target_entropy;
  t.grad_scale_B = h->B;
  t.z0_pi = h->z0[0]; t.z0_vf = h->z0[1]; t.z0_q1 = h->z0[2]; t.z0_q2 = h->z0[3]; t.z0_vt = h->z0[4];
  t.z0v_ld = h->H;
  if (h->v2.on) {     // engine v2 writes the three value heads' fc0 outputs as one [B, 3H] block
    t.z0_vf = h->v2.z0v; t.z0_q1 = h->v2.z0v + h->H; t.z0_q2 = h->v2.z0v + 2 * h->H; t.z0v_ld = 3 * h->H;
  }
  t.pi = head_w(h, "model/pi", "dense");
  t.vf = head_w(h, "model/values_fn/vf", "vf");
  t.q1 = head_w(h, "model/values_fn/qf1", "qf1");
  t.q2 = head_w(h, "model/values_fn/qf2", "qf2");
  t.vt = head_w(h, "target/values_fn/vf", "vf");
  t.ksig = h->p("model/pi/dense_1/kernel"); t.bsig = h->p("model/pi/dense_1/bias");
  t.g_pi = head_g(h, "model/pi", "dense");
  t.g_vf = head_g(h, "model/values_fn/vf", "vf");
  t.g_q1 = head_g(h, "model/values_fn/qf1", "qf1");
  t.g_q2 = head_g(h, "model/values_fn/qf2", "qf2");
  t.g_ksig = h->g("model/pi/dense_1/kernel"); t.g_bsig = h->g("model/pi/dense_1/bias");
  t.log_alpha = h->p("model/log_ent_coef"); t.g_log_alpha = h->g("model/log_ent_coef");
  t.act = h->F[1] + h->feat_dim; t.act_stride = h->FS;
  t.eps = h->eps; t.rew = h->rew_n; t.done = h->done_n;
  t.a0_pi = h->a0[0]; t.a0_vf = h->a0[1]; t.a0_q1 = h->a0[2]; t.a0_q2 = h->a0[3];
  t.dz1_pi = h->dz1[0]; t.dz1_vf = h->dz1[1]; t.dz1_q1 = h->dz1[2]; t.dz1_q2 = h->dz1[3];
  t.dz0_pi = h->dz0_pi; t.dz0_v3 = h->dz0_v3;
  if (h->v2.on) { for (int k = 0; k < 2; ++k) { t.dz0_pi_p[k] = h->v2.dz0pi[k]; t.dz0_v3_p[k] = h->v2.dz0v[k]; } }
  t.per_sample = want_per_sample ? h->per_sample : nullptr;
  t.pi_out = want_per_sample ? h->pi_out : nullptr;
  t.metrics = h->metrics;
  return t;
}

GatherArgs make_gather(b2g_sac* h, bool from_replay, bool with_next) {
  GatherArgs g{};
  g.obs = h->s_obs; g.next_obs = with_next ? h->s_next : nullptr; g.fmt = h->row_fmt;
  g.act = with_next ? h->s_act : nullptr; g.rew = h->s_rew; g.done = h->s_done;
  if (from_replay) {
    h->replay.gather_args(g, with_next);      // frames through the slots' frame indices
    g.indices = h->indices;
  }
  g.mean = h->d_mean; g.var = h->d_istd;
  g.normc = h->d_normc;
  g.B = h->B;
  g.H = h->cnn ? h->Hi : 0; g.W = h->cnn ? h->Wi : h->cfg.obs_dim; g.Cimg = h->cnn ? h->Cimg : 0;
  g.scale = h->cnn ? 255.f : 1.f;
  g.x_obs = h->x_obs; g.x_next = h->x_next;
  g.x_obs_hi = h->xp[0][0]; g.x_obs_lo = h->xp[0][1]; g.x_next_hi = h->xp[1][0]; g.x_next_lo = h->xp[1][1];
  g.F_pi = h->F[0]; g.F_v = h->F[1]; g.F_t = h->F[2]; g.FS = h->FS;
  g.feat_col = h->direct_feature() ? 512 : -1; g.act_col = h->feat_dim;
  g.rew_out = h->rew_n; g.done_out = h->done_n; g.n_act = h->A;
  return g;
}

// prep_kernel arguments: gen != 0 draws the replay slots (when the step samples) and the policy noise
PrepArgs make_prep(b2g_sac* h, unsigned long long seed, bool gen, bool apply) {
  PrepArgs pa{};
  pa.counters = h->counters; pa.step_consts = h->step_consts; pa.lr = h->d_lr; pa.metrics = h->metrics;
  pa.indices = h->indices; pa.eps = h->eps; pa.B = h->B; pa.A = h->A; pa.replay_size = nullptr;  /* device counter [5] */
  pa.ring_cap = h->cfg.buffer_capacity;
  pa.seed = seed; pa.gen = gen ? 1 : 0; pa.apply = apply ? 1 : 0;
  return pa;
}

// the ring row of one SAC step: the b2g_sac_metrics losses (sums over the ranks), log_ent_coef after the update and the
// learning rate; sac_mlog_fix turns it into what fill_metrics reports
MetricsLogSrc sac_mlog_src(b2g_sac* h) {
  MetricsLogSrc m{};
  for (int k = 0; k < 6; ++k) m.src[k] = h->metrics + MET_POLICY_LOSS + k;   // policy, qf1, qf2, value, ent_coef losses, entropy
  m.src[6] = h->p("model/log_ent_coef");
  m.src[7] = h->d_lr;
  m.K = B2G_SAC_LOG_COLS;
  return m;
}

struct Prof {
  bool on = false;
  std::vector<cudaEvent_t> ev;
  std::vector<std::string> names;
};

// Issues every launch of one gradient step on h->stream.  Returns the number of launches.
int issue_step(b2g_sac* h, bool sampled, bool apply, bool want_per_sample, Prof* prof, int* n_launch) {
  cudaStream_t s = h->stream;
  int n = 0;            // kernels (ours and, N > 1 on the NCCL path, the collective's)
  int n_copy = 0;       // memset / copy nodes: not counted as launches
  (void)n_copy;
  auto mark = [&](const char* name) {
    if (prof && prof->on) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      cudaEventRecord(e, s);
      prof->ev.push_back(e);
      prof->names.push_back(name);
    }
  };
  mark("begin");
  PrepArgs pa = make_prep(h, h->cfg.seed + 0x9E3779B97F4A7C15ull * (unsigned long long)h->cfg.rank, sampled, apply);
  // Leaf work runs on two more streams (parallel branches once captured in the step graph).  The fused launches run one
  // CTA per SM, each owning tiles near the head of its chain, so a leaf CTA still resident when one of them starts holds up
  // that whole chain: the leaf work goes where no fused launch starts.  Beside the gather, joined before fwd_fused: the
  // forward-layout weight planes and the z0 / dependency-counter zeroing (aux), the bookkeeping kernel (Adam step sizes,
  // policy noise, metric accumulators) and the gradient zeroing (aux2).  The planes get SMs only as the gather's CTAs
  // retire, so fwd_fused starts about 11 us after the gather ends (DESIGN §6).  Alongside the tail: the backward-layout
  // weight planes, joined before bwd_fused.  heads_wgrad forks after the tail and runs in the backward launch's drain.
  // Profiling (per-launch events) keeps everything serial on one stream.
  const bool fork = h->fork_leaves && !(prof && prof->on);
  cudaStream_t ax = fork ? h->aux : s;
  GatherArgs ga = make_gather(h, sampled, true);
  if (fork) {
    // the gather draws its replay slots in-kernel from prep's Philox stream, so the critical chain starts with the gather
    pa.defer_bump = 1; pa.skip_indices = 1;
    if (sampled) { ga.indices = nullptr; ga.rng_counters = h->counters; ga.seed = pa.seed; ga.indices_out = h->indices; }
    CK(cudaEventRecord(h->ev_aux[0], s));
    CK(cudaStreamWaitEvent(ax, h->ev_aux[0], 0));
    CK(cudaStreamWaitEvent(h->aux2, h->ev_aux[0], 0));
    if (h->use_planes && !h->v2.on) { planes_launch(h->d_jobs, h->n_jobs, h->job_tiles, ax); ++n; }
    if (h->v2.on) { if (int rc = v2_planes(h, false, ax)) return rc; ++n; }
    CK(cudaMemsetAsync(h->z0[0], 0, (size_t)5 * h->B * h->H * sizeof(float), ax)); ++n_copy;
    if (h->v2.on) {
      CK(cudaMemsetAsync(h->v2.z0v, 0, (size_t)3 * h->B * h->H * sizeof(float), ax)); ++n_copy;
      CK(cudaMemsetAsync(h->v2.dep_ctr, 0, (size_t)h->v2.n_dep_ctr * sizeof(int), ax)); ++n_copy;
    }
    CK(cudaEventRecord(h->ev_aux[1], ax));
    prep_launch(pa, h->aux2); ++n;
    CK(cudaMemsetAsync(h->G, 0, (size_t)(h->n_train + MET_COUNT) * sizeof(float), h->aux2)); ++n_copy;
    CK(cudaEventRecord(h->ev_aux[6], h->aux2));
  } else {
    prep_launch(pa, s); ++n; mark("prep");
  }
  if (h->v2.on) {
    if (!fork) {
      if (int rc = v2_planes(h, false, s)) return rc;
      ++n; mark("weight_planes_fwd");
      if (int rc = v2_planes(h, true, s)) return rc;
      ++n; mark("weight_planes_bwd");
    }
    if (int rc = v2_gather(h, ga, s)) return rc;
  } else gather_launch(ga, s);
  ++n; mark("gather_normalize");
  if (h->record_after_gather) CK(cudaEventRecord(h->record_after_gather, s));   // staged batch consumed
  if (fork) { CK(cudaStreamWaitEvent(s, h->ev_aux[1], 0)); CK(cudaStreamWaitEvent(s, h->ev_aux[6], 0)); }
  else {
    CK(cudaMemsetAsync(h->G, 0, (size_t)(h->n_train + MET_COUNT) * sizeof(float), s)); ++n_copy;
    CK(cudaMemsetAsync(h->z0[0], 0, (size_t)5 * h->B * h->H * sizeof(float), s)); ++n_copy;
    if (h->v2.on) { CK(cudaMemsetAsync(h->v2.z0v, 0, (size_t)3 * h->B * h->H * sizeof(float), s)); ++n_copy; }
    mark("zero_grads");
  }
  const int x3 = h->cfg.precision == B2G_PREC_BF16X3 ? 1 : 0;
  auto run_group = [&](GemmGroup& g, cudaStream_t s) -> int {
    if (g.tc) CK(gg_tc_launch(g.host.data(), (int)g.host.size(), g.total_tiles, g.host[0].flags, x3, h->num_sms, s));
    else gg_simt_launch(g.dev, (int)g.host.size(), g.total_tiles, s);
    ++n; mark(g.name.c_str());
    return 0;
  };
  if (h->v2.on) {
    if (!fork) { CK(cudaMemsetAsync(h->v2.dep_ctr, 0, (size_t)h->v2.n_dep_ctr * sizeof(int), s)); ++n_copy; }
    if (int rc = v2_launch(h, h->v2.fwd_fused[0], s)) return rc;
    ++n; mark("fwd_fused");
  } else {
    for (auto& g : h->fwd_groups) if (int rc = run_group(g, s)) return rc;
  }
  if (fork && h->v2.on) {     // the tail does not read the backward-layout planes
    CK(cudaEventRecord(h->ev_aux[7], s)); CK(cudaStreamWaitEvent(ax, h->ev_aux[7], 0));
    if (int rc = v2_planes(h, true, ax)) return rc;
    ++n;
    CK(cudaEventRecord(h->ev_aux[8], ax));
  }
  // Not launched early behind fwd_fused: its CTAs would land on the few SMs the draining persistent grid has freed, several
  // per SM, and the latency-bound tail then ended 30 us after fwd_fused instead of 18 (H100, B = 256).
  CK(tail_launch(make_tail(h, want_per_sample), s, pdl_enabled() && !h->v2.on)); ++n; mark("heads_tail");
  auto make_optim = [&]() {
    OptimArgs oa{};
    oa.P = h->P; oa.Mo = h->Mo; oa.Vo = h->Vo; oa.G = h->G; oa.T = h->P + h->n_train;
    oa.n_pi = (int)h->n_pi; oa.n_values = (int)h->n_values; oa.n_ent = (int)h->n_ent; oa.n_target = (int)h->n_target;
    oa.step_consts = h->step_consts; oa.tau = h->cfg.tau; oa.grad_scale = 1.0f / (float)h->cfg.nranks;
    oa.metrics = h->metrics; oa.apply = apply ? 1 : 0;
    return oa;
  };
  // N > 1 on engine v2: the gradients of [cnn_fc1 .. end] of both trainable blocks (+ log_ent_coef + the loss scalars: 84 % of
  // the bytes) are final after cnn_fc1's backward, so their all-reduce runs on a side stream / second communicator underneath the
  // conv backward (the GEMM grids leave ar_sms SMs to it); only the conv ranges (0.6 MB) are reduced on the critical chain.
  const bool overlap = h->overlap_ar && h->cfg.nranks > 1 && !(h->dp_p2p && apply);
  const int64_t pi_fc1 = h->tensors[h->tindex.at(h->cnn ? h->cnn_t("model/pi", 3, "w") : "model/pi/fc0/kernel")].off;
  const int64_t v_fc1 = h->tensors[h->tindex.at(h->cnn ? h->cnn_t("model/values_fn", 3, "w") : "model/values_fn/vf/fc0/kernel")].off;
  auto nccl_ck = [&](int rc) -> int {
    if (rc != 0) return b2g_fail(B2G_ENCCL, std::string("nccl: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "?"));
    return 0;
  };
  bool dp_early_opt = false;
  if (h->v2.on) {
    // backward chain on engine v2; the small head wgrads (fc0 / fc1 kernels and biases: fp32 operands) run on the CUDA cores
    // on the leaf branch.
    h->v2.sm_reserve = 0;
    cudaStream_t lx = fork ? ax : s;
    // heads_wgrad forks from the same point bwd_fused depends on.  It stays off bwd_fused's start because bwd_fused is launched
    // early (programmatic dependent launch) behind the tail and holds every SM before heads_wgrad is ready; with B2G_PDL=0
    // the two become ready together and heads_wgrad CTAs can be resident when bwd_fused places its CTAs.
    if (fork) {
      CK(cudaStreamWaitEvent(s, h->ev_aux[8], 0));    // the backward-layout planes, read from bwd_fused's first tiles on
      CK(cudaEventRecord(h->ev_aux[2], s)); CK(cudaStreamWaitEvent(ax, h->ev_aux[2], 0));
    }
    HeadsWgradArgs wa{};
    const char* hp[4] = {"model/pi", "model/values_fn/vf", "model/values_fn/qf1", "model/values_fn/qf2"};
    for (int q = 0; q < 4; ++q) {
      wa.X0[q] = h->F[q == 0 ? 0 : 1];
      wa.dz0[q] = q == 0 ? h->dz0_pi : h->dz0_v3 + (q - 1) * h->H;
      wa.dz0_ld[q] = q == 0 ? h->H : 3 * h->H;
      wa.a0[q] = h->a0[q]; wa.dz1[q] = h->dz1[q];
      wa.M0[q] = q >= 2 ? h->feat_dim + h->A : h->feat_dim;
      wa.g_k0[q] = h->g(std::string(hp[q]) + "/fc0/kernel"); wa.g_b0[q] = h->g(std::string(hp[q]) + "/fc0/bias");
      wa.g_k1[q] = h->g(h->fc1(hp[q]) + "/kernel"); wa.g_b1[q] = h->g(h->fc1(hp[q]) + "/bias");
    }
    wa.x0_ld = h->FS; wa.B = h->B; wa.H = h->H;
    heads_wgrad_launch(wa, lx); ++n; if (!fork) mark("heads_wgrad");
    // single GPU: the chain heads_dgrad .. conv wgrads is one fused launch.  Overlapped all-reduce: two (cut after cnn_fc1, where
    // the early all-reduce starts).
    if (!overlap) {
      if (int rc = v2_launch(h, h->v2.bwd_fused[0], s)) return rc;
      ++n; mark("bwd_fused");
    } else {
      if (int rc = v2_launch(h, h->v2.bwd_fused[1], s)) return rc;
      ++n; mark("bwd_fused_fc");
      CK(cudaMemcpyAsync(h->G + h->n_train, h->metrics, MET_GN_PI * sizeof(float), cudaMemcpyDeviceToDevice, s)); ++n_copy;
      CK(cudaEventRecord(h->ev_fork, s));
      CK(cudaStreamWaitEvent(h->side, h->ev_fork, 0));
      if (fork) { CK(cudaEventRecord(h->ev_aux[4], ax)); CK(cudaStreamWaitEvent(h->side, h->ev_aux[4], 0)); }   // heads_wgrad
      if (int rc = nccl_ck(g_nccl.GroupStart())) return rc;
      if (int rc = nccl_ck(g_nccl.AllReduce(h->G + pi_fc1, h->G + pi_fc1, (size_t)(h->n_pi - pi_fc1), 7, 0, h->nccl_comm2, h->side))) return rc;
      if (int rc = nccl_ck(g_nccl.AllReduce(h->G + v_fc1, h->G + v_fc1, (size_t)(h->n_train + MET_COUNT - v_fc1), 7, 0, h->nccl_comm2, h->side))) return rc;
      if (int rc = nccl_ck(g_nccl.GroupEnd())) return rc;
      ++n;
      if ((pi_fc1 & 3) == 0 && (v_fc1 & 3) == 0 && (h->n_pi & 3) == 0) {
        // the reduced ranges get their Adam / Polyak pass right behind the collective, still underneath the conv backward; the
        // closing optimiser launch only sweeps the conv kernels (after the late, 0.6 MB all-reduce)
        OptimArgs oe = make_optim();
        oe.r_lo[0] = (int)pi_fc1; oe.r_hi[0] = (int)h->n_pi;
        oe.r_lo[1] = (int)v_fc1; oe.r_hi[1] = (int)(h->n_pi + h->n_values + h->n_ent);
        optim_launch(oe, h->side); ++n;
        dp_early_opt = true;
      }
      CK(cudaEventRecord(h->ev_join, h->side));
      h->v2.sm_reserve = h->ar_sms;
      if (int rc = v2_launch(h, h->v2.bwd_fused[2], s)) return rc;
      ++n; mark("bwd_fused_conv");
    }
    h->v2.sm_reserve = 0;
  } else {
    // index of the last backward group that touches cnn_fc1 / the heads: the cnn_fc1 bias sums can start behind it
    int last_fc1 = -1;
    for (size_t i = 0; i < h->bwd_groups.size(); ++i)
      if (h->bwd_groups[i].name.find("fc1") != std::string::npos || h->bwd_groups[i].name.find("heads") != std::string::npos) last_fc1 = (int)i;
    for (size_t i = 0; i < h->bwd_groups.size(); ++i) {
      const bool leaf = fork && h->bwd_groups[i].name == "heads_wgrad";
      if (fork && h->use_planes && i + 1 == h->bwd_groups.size()) {
        // every gradient map the conv bias sums read exists once the next-to-last group (conv2_bwd) is issued:
        // the sums overlap conv1_wgrad
        CK(cudaEventRecord(h->ev_aux[4], s)); CK(cudaStreamWaitEvent(ax, h->ev_aux[4], 0));
        colsum_launch(h->d_colsum, h->n_colsum, h->colsum_ctas, ax); ++n;
      }
      if (leaf) {           // consumes only what the tail wrote; nothing downstream but the optimiser reads its output
        CK(cudaEventRecord(h->ev_aux[2], s));
        CK(cudaStreamWaitEvent(ax, h->ev_aux[2], 0));
      }
      if (int rc = run_group(h->bwd_groups[i], leaf ? ax : s)) return rc;
      if ((int)i == last_fc1) {
        if (fork) { CK(cudaEventRecord(h->ev_aux[3], s)); CK(cudaStreamWaitEvent(ax, h->ev_aux[3], 0)); }
        if (h->use_planes && h->n_colsum_early) {
          colsum_launch(h->d_colsum_early, h->n_colsum_early, h->colsum_early_ctas, ax); ++n; mark("bias_grads_fc1");
        }
      }
    }
    if (h->use_planes && !fork) { colsum_launch(h->d_colsum, h->n_colsum, h->colsum_ctas, s); ++n; mark("bias_grads"); }
  }
  if (fork) { CK(cudaEventRecord(h->ev_aux[5], ax)); CK(cudaStreamWaitEvent(s, h->ev_aux[5], 0)); }
  if (h->cfg.nranks > 1 && !(h->dp_p2p && apply)) {
    if (overlap) {
      // late all-reduce: the conv gradients of both blocks (0.29 MB each), then join the early one
      if (int rc = nccl_ck(g_nccl.GroupStart())) return rc;
      if (int rc = nccl_ck(g_nccl.AllReduce(h->G, h->G, (size_t)pi_fc1, 7, 0, h->nccl_comm, s))) return rc;
      if (int rc = nccl_ck(g_nccl.AllReduce(h->G + h->n_pi, h->G + h->n_pi, (size_t)(v_fc1 - h->n_pi), 7, 0, h->nccl_comm, s))) return rc;
      if (int rc = nccl_ck(g_nccl.GroupEnd())) return rc;
      ++n;
      CK(cudaStreamWaitEvent(s, h->ev_join, 0));
    } else {
      // losses/means ride behind the gradients in the same buffer
      CK(cudaMemcpyAsync(h->G + h->n_train, h->metrics, MET_GN_PI * sizeof(float), cudaMemcpyDeviceToDevice, s)); ++n_copy;
      if (int rc = nccl_ck(g_nccl.AllReduce(h->G, h->G, (size_t)(h->n_train + MET_COUNT), /*ncclFloat32*/ 7, /*ncclSum*/ 0, h->nccl_comm, s))) return rc;
      ++n;
    }
    CK(cudaMemcpyAsync(h->metrics, h->G + h->n_train, MET_GN_PI * sizeof(float), cudaMemcpyDeviceToDevice, s)); ++n_copy;
    mark("allreduce");
  }
  OptimArgs oa = make_optim();
  oa.bump_counter = (fork && sampled) ? h->counters + 4 : nullptr;
  if (dp_early_opt) {
    oa.r_lo[0] = 0; oa.r_hi[0] = (int)pi_fc1;
    oa.r_lo[1] = (int)h->n_pi; oa.r_hi[1] = (int)v_fc1;
  }
  if (h->dp_p2p && apply) {
    // the optimiser launch is the collective (common.cuh: DpArgs); it also sums the loss scalars across the ranks
    DpArgs da{};
    da.o = oa; da.rank = h->cfg.rank; da.nranks = h->cfg.nranks;
    for (int q = 0; q < h->cfg.nranks; ++q) { da.R_peer[q] = h->dp_G[q]; da.P_peer[q] = h->dp_P[q]; da.x_peer[q] = h->dp_X[q]; }
    da.counters = h->counters; da.sync = h->dp_sync;
    for (int k = 0; k < 2; ++k) { da.skip_lo4[k] = h->dp_skip[k][0]; da.skip_hi4[k] = h->dp_skip[k][1]; }
    dp_optim_launch(da, h->num_sms, s); ++n;
    mark("adam_polyak_dp");
  } else {     // (a gradient-only step of a connected learner takes the NCCL path above)
    optim_launch(oa, s); ++n; mark("adam_polyak");
  }
  if (h->mlog.on() && apply) {     // behind every write of the step's losses, log_ent_coef's update included
    mlog_append(h->mlog, sac_mlog_src(h), h->counters + 3, s); ++n; mark("metrics_log");
  }
  if (h->use_planes && apply && !h->v2.on) {
    // with fork: refreshed on the aux branch at the head of the next step (the API entry points mark them stale)
    if (!fork) { planes_launch(h->d_jobs, h->n_jobs, h->job_tiles, s); ++n; mark("weight_planes"); }
  }
  CK(cudaGetLastError());
  if (n_launch) *n_launch = n;
  return 0;
}

// BF16 planes of the CNN weights follow every optimiser step inside the step itself; after a host upload
// (b2g_set_param) they are refreshed here, outside any graph.
void refresh_planes(b2g_sac* h, bool for_step = false) {
  if (for_step && (h->fork_leaves || h->v2.on)) {     // the step refreshes the planes itself and leaves them one update behind
    h->planes_dirty = true;
    return;
  }
  if (h->use_planes && h->planes_dirty) {
    planes_launch(h->d_jobs, h->n_jobs, h->job_tiles, h->stream);
    h->planes_dirty = false;
  }
}

void fill_metrics(const b2g_sac* h, const float* m, const long long* cnt, b2g_sac_metrics* out) {
  const float inv = 1.0f / (float)h->cfg.nranks;
  out->policy_loss = m[MET_POLICY_LOSS] * inv; out->qf1_loss = m[MET_QF1_LOSS] * inv; out->qf2_loss = m[MET_QF2_LOSS] * inv;
  out->value_loss = m[MET_VALUE_LOSS] * inv; out->ent_coef_loss = m[MET_ENT_COEF_LOSS] * inv; out->entropy = m[MET_ENTROPY] * inv;
  out->mean_q1 = m[MET_MEAN_Q1] * inv; out->mean_q2 = m[MET_MEAN_Q2] * inv; out->mean_v = m[MET_MEAN_V] * inv;
  out->mean_logp = m[MET_MEAN_LOGP] * inv;
  out->grad_norm_pi = sqrtf(m[MET_GN_PI]); out->grad_norm_values = sqrtf(m[MET_GN_VALUES]);
  out->grad_ent = m[MET_COUNT + 1] * inv;
  out->ent_coef = expf(m[MET_COUNT]);     // value AFTER the update when apply_update != 0 (SB logs the pre-update value)
  out->n_updates = cnt[3];
}

// the step's metrics -> pinned met[MET_COUNT + 2] (the accumulators, then log_alpha and its gradient) and cnt[8], in stream order
int copy_metrics_async(b2g_sac* h, float* met, long long* cnt) {
  CK(cudaMemcpyAsync(met, h->metrics, MET_COUNT * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(met + MET_COUNT, h->p("model/log_ent_coef"), sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(met + MET_COUNT + 1, h->g("model/log_ent_coef"), sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(cnt, h->counters, 8 * sizeof(long long), cudaMemcpyDeviceToHost, h->stream));
  return 0;
}

int fetch_metrics(b2g_sac* h, b2g_sac_metrics* out) {
  if (int rc = copy_metrics_async(h, h->h_met, h->h_cnt)) return rc;
  CK(cudaStreamSynchronize(h->stream));
  if (out) fill_metrics(h, h->h_met, h->h_cnt, out);
  return 0;
}

int find_tensor(const b2g_sac* h, const char* name) {
  if (!name) return -1;
  std::string n(name);
  if (n.size() > 2 && n.compare(n.size() - 2, 2, ":0") == 0) n.resize(n.size() - 2);
  auto it = h->tindex.find(n);
  return it == h->tindex.end() ? -1 : it->second;
}

// element of a caller's observation that element e of a ring row holds; -1 for the pads of a compact row
int full_index(const b2g_sac* h, int e) {
  if (!h->cnn) return e;
  const int Ci = h->Cimg, npx = h->Hi * h->Wi * Ci;
  if (e < npx) return (e / Ci) * h->Cobs + e % Ci;
  return e == npx && h->direct_feature() ? Ci : -1;
}

// n caller observations (host or device memory) -> rows (first + i) % wrap of dst in the ring layout, on h->stream.  CNN: copied in
// pieces through the full-layout staging buffer and compacted (stream order frees the buffer for the next piece); MLP: a plain
// copy, for which first + n <= wrap.
int load_rows(b2g_sac* h, const float* src, float* dst, long long first, long long wrap, long long n) {
  const size_t E = h->E;
  if (!h->cnn) {
    CK(cudaMemcpyAsync(dst + first * E, src, n * E * sizeof(float), cudaMemcpyDefault, h->stream));
    return 0;
  }
  for (long long i = 0; i < n; i += h->stage_rows) {
    const int m = (int)std::min<long long>(h->stage_rows, n - i);
    CK(cudaMemcpyAsync(h->obs_stage, src + i * E, m * E * sizeof(float), cudaMemcpyDefault, h->stream));
    compact_rows(h->obs_stage, dst, first + i, wrap, m, h->Hi * h->Wi, h->Cimg, h->Cobs, h->stream);
  }
  return 0;
}

}  // namespace

// ================================================================================================
// hooks of the observe path (obsnorm.cu; contracts in sac_internal.cuh)
// ================================================================================================
namespace b2g {

int sac_act_rows(b2g_sac* h, const float* rows, int chunk, int deterministic) {
  refresh_planes(h);
  prep_launch(make_prep(h, h->cfg.seed ^ 0xA5A5A5A5DEADBEEFull, !deterministic, false), h->stream);
  GatherArgs g = make_gather(h, false, false);
  g.obs = rows;
  gather_launch(g, h->stream);
  for (auto& gr : h->act_groups) {
    if (gr.tc) CK(gg_tc_launch(gr.host.data(), (int)gr.host.size(), gr.total_tiles, gr.host[0].flags, h->cfg.precision == B2G_PREC_BF16X3 ? 1 : 0, h->num_sms, h->stream));
    else gg_simt_launch(gr.dev, (int)gr.host.size(), gr.total_tiles, h->stream);
  }
  CK(b2g::act_launch(make_tail(h, false), chunk, deterministic, h->pi_out, h->stream));
  return 0;
}

}  // namespace b2g

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" {

int b2g_sac_dp_export(b2g_sac* h, void* out192) {
  B2G_USABLE(h);
  if (!h || !out192) return b2g_fail(B2G_EINVAL, "b2g_sac_dp_export: null argument");
  cudaSetDevice(h->cfg.device);
  if (!h->dp_x) {
    if (int rc = dev_alloc(h->allocs, h->stream, &h->dp_x, 256)) return rc;
    if (int rc = dev_alloc(h->allocs, h->stream, &h->dp_recv, h->n_train + 64 * DP_MAX_RANKS)) return rc;      // [src rank][my slice], slices <= ceil(n/N) + pad
    if (int rc = dev_alloc(h->allocs, h->stream, &h->dp_sync, 64)) return rc;
    CK(cudaStreamSynchronize(h->stream));
  }
  cudaIpcMemHandle_t hd[3];
  CK(cudaIpcGetMemHandle(&hd[0], h->P));
  CK(cudaIpcGetMemHandle(&hd[1], h->dp_recv));
  CK(cudaIpcGetMemHandle(&hd[2], h->dp_x));
  static_assert(sizeof(hd) == B2G_DP_EXPORT_BYTES, "export blob size");
  memcpy(out192, hd, sizeof(hd));
  return 0;
}

int b2g_debug_dp_stamps(b2g_sac* h, long long* out5) {     /* bring-up: phase timestamps of the last peer-memory optimiser launch */
  if (!h || !h->dp_sync) return b2g_fail(B2G_EINVAL, "b2g_debug_dp_stamps: not connected");
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaMemcpy(out5, h->dp_sync + 8, 5 * sizeof(long long), cudaMemcpyDeviceToHost));
  return 0;
}

int b2g_sac_dp_connect(b2g_sac* h, const void* all_exports, int nranks) {
  B2G_USABLE(h);
  if (!h || !all_exports) return b2g_fail(B2G_EINVAL, "b2g_sac_dp_connect: null argument");
  if (nranks != h->cfg.nranks || nranks < 2 || nranks > DP_MAX_RANKS) return b2g_fail(B2G_EINVAL, "b2g_sac_dp_connect: nranks must equal the learner's (2..8)");
  if (!h->dp_x) return b2g_fail(B2G_EINVAL, "b2g_sac_dp_connect: call b2g_sac_dp_export first");
  if (h->dp_p2p) return b2g_fail(B2G_ESTATE, "b2g_sac_dp_connect: already connected");
  if (((h->n_pi | h->n_values | h->n_ent | h->n_target) & 3) != 0) return b2g_fail(B2G_EINVAL, "b2g_sac_dp_connect: arena segments are not float4 aligned");
  cudaSetDevice(h->cfg.device);
  CK(cudaStreamSynchronize(h->stream));
  for (int q = 0; q < nranks; ++q) {
    if (q == h->cfg.rank) { h->dp_P[q] = h->P; h->dp_G[q] = h->dp_recv; h->dp_X[q] = h->dp_x; continue; }
    cudaIpcMemHandle_t hd[3];
    memcpy(hd, (const char*)all_exports + (size_t)q * B2G_DP_EXPORT_BYTES, sizeof(hd));
    void* p[3] = {nullptr, nullptr, nullptr};
    for (int k = 0; k < 3; ++k) {
      CK(cudaIpcOpenMemHandle(&p[k], hd[k], cudaIpcMemLazyEnablePeerAccess));
      h->dp_opened.push_back(p[k]);
    }
    h->dp_P[q] = (float*)p[0]; h->dp_G[q] = (float*)p[1]; h->dp_X[q] = (int*)p[2];
  }
  // the cnn_fc1 weight gradients (80 % of the gradient bytes) are final when their tiles are stored: their epilogues push them
  h->dp_skip[0][0] = h->dp_skip[0][1] = h->dp_skip[1][0] = h->dp_skip[1][1] = 0;
  if (h->v2.on) {
    const int n_train4 = (int)((h->n_pi + h->n_values + h->n_ent) >> 2), per4 = (n_train4 + nranks - 1) / nranks;
    const std::string names[2] = {h->cnn_t("model/pi", 3, "w"), h->cnn_t("model/values_fn", 3, "w")};
    for (int k = 0; k < 2; ++k) {
      const float* gp = h->g(names[k]);
      const auto& t = h->tensors[h->tindex.at(names[k])];
      bool found = false;
      auto patch = [&](std::vector<CgGroup>& groups) {
        for (CgGroup& g : groups)
          for (int i = 0; i < g.n; ++i) {
            CgProblem& P = g.host[i];
            if (P.epi != CG_EPI_WGRAD || P.atomic || P.out_f != gp) continue;
            for (int q = 0; q < nranks; ++q) P.dp_recv[q] = h->dp_G[q];
            P.dp_gbase = h->G; P.dp_rank = h->cfg.rank; P.dp_n = nranks; P.dp_per4 = per4;
            found = true;
          }
      };
      patch(h->v2.bwd_fused);
      if (found && (t.off & 3) == 0) { h->dp_skip[k][0] = (int)(t.off >> 2); h->dp_skip[k][1] = (int)((t.off + 1024 * 512) >> 2); }
    }
  }
  h->dp_p2p = true;
  if (h->graph_exec) { cudaGraphExecDestroy(h->graph_exec); h->graph_exec = nullptr; }     // the step changes shape
  for (auto& g : h->pipe_graph) if (g) { cudaGraphExecDestroy(g); g = nullptr; }
  return 0;
}

int b2g_sac_destroy(b2g_sac* h) {
  if (!h) return 0;
  cudaSetDevice(h->cfg.device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->graph_exec) cudaGraphExecDestroy(h->graph_exec);
  for (auto& g : h->pipe_graph) if (g) cudaGraphExecDestroy(g);
  for (void* q : h->dp_opened) cudaIpcCloseMemHandle(q);
  nccl_comm_destroy(h->nccl_comm2);
  nccl_comm_destroy(h->nccl_comm);
  if (h->side) cudaStreamDestroy(h->side);
  if (h->aux) { cudaStreamSynchronize(h->aux); cudaStreamDestroy(h->aux); }
  if (h->aux2) { cudaStreamSynchronize(h->aux2); cudaStreamDestroy(h->aux2); }
  for (auto& e : h->ev_aux) if (e) cudaEventDestroy(e);
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  if (h->ev_join) cudaEventDestroy(h->ev_join);
  enc_stage_destroy(h->rms.enc);
  for (void* q : h->allocs) cudaFree(q);
  for (int q = 0; q < 2; ++q) { if (h->hc_obs[q]) cudaFreeHost(h->hc_obs[q]); if (h->hc_next[q]) cudaFreeHost(h->hc_next[q]); }
  if (h->h_met) cudaFreeHost(h->h_met);
  if (h->h_cnt) cudaFreeHost(h->h_cnt);
  h->replay.release();
  for (int k = 0; k < 2; ++k) { if (h->hp_stats[k]) cudaFreeHost(h->hp_stats[k]); if (h->ev_stats[k]) cudaEventDestroy(h->ev_stats[k]); }
  for (int j = 0; j < 2; ++j) {
    if (h->ev_h2d[j]) cudaEventDestroy(h->ev_h2d[j]);
    if (h->ev_consumed[j]) cudaEventDestroy(h->ev_consumed[j]);
    if (h->ev_met[j]) cudaEventDestroy(h->ev_met[j]);
    if (h->pm_met[j]) cudaFreeHost(h->pm_met[j]);
    if (h->pm_cnt[j]) cudaFreeHost(h->pm_cnt[j]);
  }
  mlog_free(&h->mlog);
  if (h->cstream) cudaStreamDestroy(h->cstream);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

int b2g_sac_create(const b2g_sac_cfg* cfg, b2g_sac** out) { return b2g_sac_create2(cfg, nullptr, out); }

int b2g_sac_create2(const b2g_sac_cfg* cfg, const b2g_replay_cfg* replay, b2g_sac** out) {
  return b2g_sac_create3(cfg, replay, nullptr, out);
}

int b2g_sac_create3(const b2g_sac_cfg* cfg, const b2g_replay_cfg* replay, const b2g_sac_net_cfg* net, b2g_sac** out) {
  if (!cfg || !out) return b2g_fail(B2G_EINVAL, "cfg/out is NULL");
  *out = nullptr;
  const int extractor = net ? net->extractor : B2G_CNN_AUGMENTED;
  if (extractor != B2G_CNN_AUGMENTED && extractor != B2G_CNN_NATURE)
    return b2g_fail(B2G_EINVAL, "unknown extractor (B2G_CNN_AUGMENTED or B2G_CNN_NATURE)");
  if (extractor == B2G_CNN_NATURE && cfg->obs_h <= 0)
    return b2g_fail(B2G_EINVAL, "B2G_CNN_NATURE is a CNN extractor: the MLP policy (obs_h == 0) has none");
  const bool nature = extractor == B2G_CNN_NATURE;
  const int n_img = nature ? cfg->obs_c : cfg->obs_c - 1;      // image planes conv1 reads
  if (replay && replay->u8_plane_mask && cfg->obs_h <= 0) return b2g_fail(B2G_EINVAL, "the MLP policy has no 8-bit image planes");
  if (replay && replay->u8_plane_mask && (n_img < 1 || n_img > 8 || (replay->u8_plane_mask >> n_img) != 0))
    return b2g_fail(B2G_EINVAL, nature ? "u8_plane_mask may only name image planes (below obs_c), at most 8"
                                       : "u8_plane_mask may only name image planes, at most 8 (the actuator plane is the last channel)");
  if (cfg->hidden != 64 && cfg->hidden != 128 && cfg->hidden != 192 && cfg->hidden != 256)
    return b2g_fail(B2G_EINVAL, "hidden must be 64, 128, 192 or 256 (SAC.layers [H, H])");
  if (cfg->n_act < 1 || cfg->n_act > 8) return b2g_fail(B2G_EINVAL, "n_act must be in [1,8]");
  if (cfg->batch < 1 || cfg->buffer_capacity < 1) return b2g_fail(B2G_EINVAL, "batch and buffer_capacity must be positive");
  const int64_t frame_cap = replay ? replay->frame_capacity : 2 * cfg->buffer_capacity;
  if (int rc = check_frame_capacity(frame_cap, cfg->buffer_capacity, "frame_capacity")) return rc;
  if (cfg->nranks < 1 || cfg->rank < 0 || cfg->rank >= cfg->nranks) return b2g_fail(B2G_EINVAL, "bad rank/nranks");
  if (cfg->precision < B2G_PREC_FP32_SIMT || cfg->precision > B2G_PREC_BF16)
    return b2g_fail(B2G_EINVAL, "unknown precision mode");
  int num_sms = 0;
  if (int rc = check_device(cfg->device, &num_sms)) return rc;

  b2g_sac* h = new b2g_sac();
  h->cfg = *cfg;
  h->num_sms = num_sms;
  h->cfg.nccl_id = nullptr; h->cfg.nccl_lib = nullptr;
  h->cnn = cfg->obs_h > 0;
  h->extractor = extractor;
  h->cnn_scope = kCnnScopes[nature ? 1 : 0];
  h->B = cfg->batch; h->A = cfg->n_act; h->H = cfg->hidden;
  if (h->cnn) {
    if (!nature && cfg->obs_c < 2) { delete h; return b2g_fail(B2G_EINVAL, "CNN policy needs obs_c >= 2 (image planes + feature plane)"); }
    if (nature && (cfg->obs_c < 1 || cfg->obs_c > 8)) { delete h; return b2g_fail(B2G_EINVAL, "nature_cnn needs obs_c in [1, 8]"); }
    h->Cimg = n_img; h->Cobs = cfg->obs_c; h->Hi = cfg->obs_h; h->Wi = cfg->obs_w;
    h->H1 = (h->Hi - 8) / 4 + 1; h->W1 = (h->Wi - 8) / 4 + 1;
    h->H2 = (h->H1 - 4) / 2 + 1; h->W2 = (h->W1 - 4) / 2 + 1;
    h->H3 = h->H2 - 2; h->W3 = h->W2 - 2;
    if (h->H3 * h->W3 * 64 != 1024 || (h->Wi * h->Cimg) % 4 != 0) {
      delete h;
      return b2g_fail(B2G_EINVAL, "observation size must give a 4x4x64 conv3 output (64x64 input; cnn_fc1/w is (1024,512))");
    }
    h->E = h->Hi * h->Wi * cfg->obs_c;
    h->Ec = h->Hi * h->Wi * h->Cimg + 4;
    h->feat_dim = nature ? 512 : 513;
  } else {
    if (cfg->obs_dim < 1) { delete h; return b2g_fail(B2G_EINVAL, "obs_dim must be positive for the MLP policy"); }
    h->E = h->Ec = cfg->obs_dim;
    h->feat_dim = cfg->obs_dim;
  }
  h->FS = (h->feat_dim + h->A + 7) / 8 * 8;
  auto bail = [&](int rc) { std::string keep = g_b2g_err; b2g_sac_destroy(h); g_b2g_err = keep; return rc; };
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "cudaStreamCreate failed"));
  cudaEventCreate(&h->ev0); cudaEventCreate(&h->ev1);
  build_params(h);
  int rc = 0;
  const int B = h->B;
#define DA(ptr, count) if ((rc = dev_alloc(h->allocs, h->stream, &(ptr), (size_t)(count)))) return bail(rc)
  DA(h->P, h->n_all); DA(h->Mo, h->n_train); DA(h->Vo, h->n_train); DA(h->G, h->n_train + MET_COUNT);
  DA(h->metrics, MET_COUNT); DA(h->counters, 8); DA(h->step_consts, 4); DA(h->d_lr, 1);
  const int64_t cap = cfg->buffer_capacity;
  {   // engine v2 (TMA-fed, cg.cu) trains the 64x64 CNN policy of up to 4 image channels (conv1's S layout) in the parity mode
    h->v2.on = h->cnn && cfg->precision == B2G_PREC_BF16X3 && h->Hi == 64 && h->Wi == 64 && h->Cimg <= 4;
    if (const char* dbg = getenv("B2G_CG_DEBUG")) h->v2.dbg = atoi(dbg);
  }
  h->stage_rows = std::max(B, 256);
  {   // frame formats: the fp32 compact row, and the replay frames (8-bit planes first, then the fp32 planes, then the tail)
    const int npx = h->cnn ? h->Hi * h->Wi * h->Cimg : 0, HW = h->Hi * h->Wi;
    h->row_fmt.n32 = h->Cimg; h->row_fmt.tail = 4 * npx;
    h->u8_mask = replay ? replay->u8_plane_mask : 0;
    FrameIo lay{};
    lay.fmt = h->row_fmt; lay.npx = npx; lay.Ci = h->cnn ? h->Cimg : 1; lay.Ec = h->Ec;
    lay.frame_bytes = (int64_t)h->Ec * 4;       // the compact row itself (replay_budget.frame_bytes)
    if (h->u8_mask) {
      FrameFmt& f = lay.fmt;
      f.n8 = f.n32 = 0;
      for (int c = 0; c < h->Cimg; ++c) f.ch[c] = (h->u8_mask >> c & 1) ? (signed char)f.n8++ : (signed char)(-1 - f.n32++);
      f.f32_off = HW * f.n8;
      f.tail = f.f32_off + 4 * HW * f.n32;
      if (f.f32_off % 16 != 0) return bail(b2g_fail(B2G_EINVAL, "8-bit planes need H * W * (8-bit planes) to be a multiple of 16"));
      lay.frame_bytes = (f.tail + 16 + 15) / 16 * 16;      // 16-byte frame stride: the gathers' 128-bit loads stay aligned
    }
    h->replay.frames_name = "frame_capacity";
    if ((rc = h->replay.init(h->allocs, h->stream, cap, h->E, h->A, B, false, 0.f, 0.f, frame_cap, lay, h->stage_rows))) return bail(rc);
  }
  if (h->cnn) DA(h->obs_stage, (size_t)h->stage_rows * h->E);
  DA(h->d_mean, h->Ec); DA(h->d_istd, h->Ec); DA(h->d_normc, 8);
  // obs_rms over the caller's layout; the plain nature_cnn's compact image block is the caller's observation itself: the flat table
  h->rms.E = h->E; h->rms.Cfull = h->direct_feature() ? h->Cobs : 0; h->rms.npx = h->cnn ? h->Hi * h->Wi * h->Cimg : 0;
  h->rms.d_mean = h->d_mean; h->rms.d_istd = h->d_istd; h->rms.set_call = "b2g_obs_rms_set";
  for (int k = 0; k < 2; ++k) {
    if (cudaMallocHost((void**)&h->hp_stats[k], (size_t)(2 * h->Ec + 8) * sizeof(double)) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->ev_stats[k], cudaEventDisableTiming) != cudaSuccess)
      return bail(b2g_fail(B2G_ECUDA, "norm-stat staging"));
  }
  DA(h->s_obs, (size_t)B * h->Ec); DA(h->s_next, (size_t)B * h->Ec); DA(h->s_act, B * h->A); DA(h->s_rew, B); DA(h->s_done, B);
  if (h->cnn) {
    DA(h->x_obs, (size_t)B * h->Hi * h->Wi * h->Cimg); DA(h->x_next, (size_t)B * h->Hi * h->Wi * h->Cimg);
    for (int n = 0; n < 3; ++n) {
      DA(h->h1[n], (size_t)B * h->H1 * h->W1 * 32); DA(h->h2[n], (size_t)B * h->H2 * h->W2 * 64); DA(h->h3[n], (size_t)B * 1024);
    }
    for (int n = 0; n < 2 && !h->v2.on; ++n) {     // gradient maps of the round-1 backward
      DA(h->dZ4[n], (size_t)B * 512); DA(h->dZ3p[n], (size_t)B * (h->H3 + 4) * (h->W3 + 4) * 64);
      DA(h->dZ2p[n], (size_t)B * (h->H2 + 3) * (h->W2 + 3) * 64); DA(h->dZ1[n], (size_t)B * h->H1 * h->W1 * 32);
    }
  }
  h->use_planes = h->cnn && cfg->precision != B2G_PREC_FP32_SIMT;
  if (h->v2.on && (rc = v2_alloc(h))) return bail(rc);
  if (h->use_planes) {
    const size_t nx = (size_t)B * h->Hi * h->Wi * h->Cimg;
    for (int k = 0; k < 2; ++k) { DA(h->xp[0][k], nx); DA(h->xp[1][k], nx); }
    for (int n = 0; n < 3; ++n)
      for (int k = 0; k < 2; ++k) {
        if (h->v2.on) {      // policy inference writes its hi / lo activation planes into planes 0 / 1 of the v2 activations
          h->h1p[n][k] = h->v2.H1[n][k]; h->h2p[n][k] = h->v2.H2[n][k]; h->h3p[n][k] = h->v2.H3[n][k];
          continue;
        }
        DA(h->h1p[n][k], (size_t)B * h->H1 * h->W1 * 32); DA(h->h2p[n][k], (size_t)B * h->H2 * h->W2 * 64); DA(h->h3p[n][k], (size_t)B * 1024);
      }
    for (int n = 0; n < 2 && !h->v2.on; ++n)
      for (int k = 0; k < 2; ++k) {
        DA(h->dZ4p[n][k], (size_t)B * 512); DA(h->dZ3pp[n][k], (size_t)B * (h->H3 + 4) * (h->W3 + 4) * 64);
        DA(h->dZ2pp[n][k], (size_t)B * (h->H2 + 3) * (h->W2 + 3) * 64);
        DA(h->dZ1p[n][k], (size_t)B * h->H1 * h->W1 * 32);
      }
    const size_t wsz[4] = {(size_t)64 * h->Cimg * 32, 512 * 64, 576 * 64, 1024 * 512};
    for (int n = 0; n < 3; ++n)
      for (int l = 0; l < 4; ++l)
        for (int k = 0; k < 4; ++k) {
          if (n == 2 && k < 2) continue;      // the target network only runs forward: transposed planes suffice
          DA(h->wp[n][l][k], wsz[l]);
        }
  }
  for (int n = 0; n < 3; ++n) DA(h->F[n], (size_t)B * h->FS);
  DA(h->z0[0], 5 * B * h->H);                      // one block: zeroed with a single memset per step
  for (int q = 1; q < 5; ++q) h->z0[q] = h->z0[0] + (size_t)q * B * h->H;
  for (int q = 0; q < 4; ++q) { DA(h->a0[q], B * h->H); DA(h->dz1[q], B * h->H); }
  DA(h->dz0_pi, B * h->H); DA(h->dz0_v3, B * 3 * h->H);
  DA(h->per_sample, 7 * B); DA(h->pi_out, B * h->A); DA(h->eps, B * h->A + 4); DA(h->rew_n, B); DA(h->done_n, B);
  DA(h->indices, B + 4);
#undef DA
  if (cudaMallocHost((void**)&h->h_met, (MET_COUNT + 2) * sizeof(float)) != cudaSuccess ||
      cudaMallocHost((void**)&h->h_cnt, 8 * sizeof(long long)) != cudaSuccess)
    return bail(b2g_fail(B2G_ECUDA, "cudaMallocHost failed"));
  for (int j = 0; j < 2; ++j) {
    if ((rc = dev_alloc(h->allocs, h->stream, &h->ps_obs[j], (size_t)B * h->Ec)) || (rc = dev_alloc(h->allocs, h->stream, &h->ps_next[j], (size_t)B * h->Ec))) return bail(rc);
    if (cudaEventCreateWithFlags(&h->ev_h2d[j], cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->ev_consumed[j], cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->ev_met[j], cudaEventDisableTiming) != cudaSuccess ||
        cudaMallocHost((void**)&h->pm_met[j], (MET_COUNT + 2) * sizeof(float)) != cudaSuccess ||
        cudaMallocHost((void**)&h->pm_cnt[j], 8 * sizeof(long long)) != cudaSuccess)
      return bail(b2g_fail(B2G_ECUDA, "pipelined-path resources"));
  }
  if (cudaStreamCreateWithFlags(&h->cstream, cudaStreamNonBlocking) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "copy stream"));
  {   // leaf branch of the step (B2G_FORK=0 keeps the step on one stream)
    const char* fk = getenv("B2G_FORK");
    if (!(fk && atoi(fk) == 0)) {
      if (cudaStreamCreateWithFlags(&h->aux, cudaStreamNonBlocking) != cudaSuccess ||
          cudaStreamCreateWithFlags(&h->aux2, cudaStreamNonBlocking) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "aux stream"));
      for (auto& e : h->ev_aux)
        if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "aux events"));
      h->fork_leaves = true;
    }
  }
  // identity normalisation until b2g_set_norm_stats is called
  {
    std::vector<double> ones(h->Ec, 1.0);
    if (cudaMemcpyAsync(h->d_istd, ones.data(), h->Ec * sizeof(double), cudaMemcpyHostToDevice, h->stream) != cudaSuccess ||
        cudaStreamSynchronize(h->stream) != cudaSuccess)
      return bail(b2g_fail(B2G_ECUDA, "init copy failed"));
  }
  if ((rc = build_groups(h))) return bail(rc);
  if (h->v2.on && (rc = v2_create(h))) return bail(rc);
  if (cfg->nranks > 1) {
    if (!cfg->nccl_id) return bail(b2g_fail(B2G_EINVAL, "nranks > 1 needs nccl_id"));
    if ((rc = nccl_comm_init(&h->nccl_comm, cfg->nranks, cfg->nccl_id, cfg->rank, cfg->nccl_lib))) return bail(rc);
    {   // second communicator + side stream for the early (overlapped) all-reduce
      // engine v2 only (B2G_AR_OVERLAP=0 puts the whole all-reduce back on the critical chain)
      const char* ov = getenv("B2G_AR_OVERLAP");
      const bool want_ov = h->v2.on && !(ov && ov[0] == '0');
      if (want_ov && g_nccl.CommSplit && g_nccl.GroupStart && g_nccl.GroupEnd) {
        if (g_nccl.CommSplit(h->nccl_comm, 0, cfg->rank, &h->nccl_comm2, nullptr) == 0 && h->nccl_comm2 &&
            cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking) == cudaSuccess &&
            cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming) == cudaSuccess) {
          h->overlap_ar = true;
          if (const char* e = getenv("B2G_AR_SMS")) h->ar_sms = atoi(e);
          g_nccl.AllReduce(h->G, h->G, 1024, 7, 0, h->nccl_comm2, h->side);     // warm-up
          cudaStreamSynchronize(h->side);
        }
      }
    }
    // warm the communicator up outside any stream capture (NCCL allocates its channels lazily)
    const int nrc = g_nccl.AllReduce(h->G, h->G, (size_t)(h->n_train + MET_COUNT), 7, 0, h->nccl_comm, h->stream);
    if (nrc != 0 || cudaStreamSynchronize(h->stream) != cudaSuccess) return bail(b2g_fail(B2G_ENCCL, "NCCL warm-up all-reduce failed"));
  }
  const char* ng = getenv("B2G_NO_GRAPH");
  h->use_graph = !(ng && ng[0] == '1');
  if (cudaStreamSynchronize(h->stream) != cudaSuccess) return bail(b2g_fail(B2G_ECUDA, "create: sync failed"));
  *out = h;
  return 0;
}

int b2g_sync(b2g_sac* h) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}

int b2g_param_count(const b2g_sac* h) { B2G_USABLE(h); return h ? (int)h->tensors.size() : 0; }

int b2g_param_info(const b2g_sac* h, int idx, const char** name, int64_t* numel, int32_t* ndim, int64_t shape[4]) {
  B2G_USABLE(h);
  if (!h || idx < 0 || idx >= (int)h->tensors.size()) return b2g_fail(B2G_EINVAL, "bad tensor index");
  const Tensor& t = h->tensors[idx];
  if (name) *name = t.name.c_str();
  if (numel) *numel = t.numel;
  if (ndim) *ndim = t.ndim;
  if (shape) for (int i = 0; i < 4; ++i) shape[i] = t.shape[i];
  return 0;
}

static int copy_tensor(b2g_sac* h, const char* name, float* arena, float* host, size_t numel, bool to_host, bool trainable_only) {
  if (!h || !host) return b2g_fail(B2G_EINVAL, "NULL argument");
  const int i = find_tensor(h, name);
  if (i < 0) return b2g_fail(B2G_EINVAL, std::string("unknown variable: ") + (name ? name : "(null)"));
  const Tensor& t = h->tensors[i];
  if ((int64_t)numel != t.numel) return b2g_fail(B2G_EINVAL, std::string("size mismatch for ") + t.name);
  if (trainable_only && t.group == 3) return b2g_fail(B2G_EINVAL, std::string("not a trainable variable: ") + t.name);
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  if (to_host) CK(cudaMemcpy(host, arena + t.off, numel * sizeof(float), cudaMemcpyDeviceToHost));
  else CK(cudaMemcpy(arena + t.off, host, numel * sizeof(float), cudaMemcpyHostToDevice));
  return 0;
}

int b2g_get_param(b2g_sac* h, const char* name, float* dst, size_t numel) { B2G_USABLE(h); return copy_tensor(h, name, h ? h->P : nullptr, dst, numel, true, false); }
int b2g_set_param(b2g_sac* h, const char* name, const float* src, size_t numel) {
  B2G_USABLE(h);
  int rc = copy_tensor(h, name, h ? h->P : nullptr, const_cast<float*>(src), numel, false, false);
  if (rc == 0) h->planes_dirty = true;
  return rc;
}
int b2g_get_grad(b2g_sac* h, const char* name, float* dst, size_t numel) {
  B2G_USABLE(h);
  int rc = copy_tensor(h, name, h ? h->G : nullptr, dst, numel, true, true);
  if (rc == 0 && h->cfg.nranks > 1) for (size_t i = 0; i < numel; ++i) dst[i] /= (float)h->cfg.nranks;
  return rc;
}
int b2g_get_adam(b2g_sac* h, const char* name, float* m, float* v, size_t numel) {
  B2G_USABLE(h);
  if (int rc = copy_tensor(h, name, h ? h->Mo : nullptr, m, numel, true, true)) return rc;
  return copy_tensor(h, name, h->Vo, v, numel, true, true);
}
int b2g_reset_optimizer(b2g_sac* h) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemsetAsync(h->Mo, 0, h->n_train * sizeof(float), h->stream));
  CK(cudaMemsetAsync(h->Vo, 0, h->n_train * sizeof(float), h->stream));
  CK(cudaMemsetAsync(h->counters, 0, 4 * sizeof(long long), h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}

int b2g_replay_add(b2g_sac* h, const float* obs, const float* act, const float* rew, const float* next_obs, const float* done,
                   int64_t n) {
  B2G_USABLE(h);
  if (!h || !obs || !act || !rew || !next_obs || !done || n < 0) return b2g_fail(B2G_EINVAL, "NULL argument");
  CK(cudaSetDevice(h->cfg.device));
  auto load = [h](const float* src, float* dst, int m) { return load_rows(h, src, dst, 0, h->stage_rows, m); };
  if (int rc = h->replay.add(obs, act, rew, next_obs, done, n, h->counters, h->stream, load)) return rc;
  h->rms.up_other += (int64_t)(n * (2 * h->E + h->A + 2) * sizeof(float));
  return 0;
}

int64_t b2g_replay_size(const b2g_sac* h) { B2G_USABLE(h); return h ? h->replay.size : 0; }

int b2g_replay_info(const b2g_sac* h, int64_t* capacity, int64_t* size, int64_t* frame_capacity, int64_t* live_frames,
                    int64_t* bytes, int64_t* evicted_early) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  h->replay.info(capacity, size, frame_capacity, live_frames, bytes, evicted_early);
  return 0;
}

int b2g_replay_get(b2g_sac* h, int64_t slot, float* obs, float* act, float* rew, float* next_obs, float* done) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  std::vector<float> row[2] = {std::vector<float>(obs ? h->Ec : 0), std::vector<float>(next_obs ? h->Ec : 0)};
  if (int rc = h->replay.get(slot, obs ? row[0].data() : nullptr, act, rew, next_obs ? row[1].data() : nullptr, done, nullptr,
                             h->cfg.device, h->stream))
    return rc;
  // the caller's layout: for the CNN policy the actuator plane comes back as zeros except pixel [0,0] (all the policy reads of it)
  for (int w = 0; w < 2; ++w) {
    float* dst = w ? next_obs : obs;
    if (!dst) continue;
    std::fill(dst, dst + h->E, 0.f);
    for (int e = 0; e < h->Ec; ++e)
      if (const int f = full_index(h, e); f >= 0) dst[f] = row[w][e];
  }
  return 0;
}

int b2g_get_last_batch(b2g_sac* h, int32_t* indices, float* eps, float* per_sample, float* pi_out) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  const size_t B = h->B, A = h->A;
  if (indices) CK(cudaMemcpy(indices, h->indices, B * sizeof(int32_t), cudaMemcpyDeviceToHost));
  if (eps) CK(cudaMemcpy(eps, h->eps, B * A * sizeof(float), cudaMemcpyDeviceToHost));
  if (per_sample) CK(cudaMemcpy(per_sample, h->per_sample, 7 * B * sizeof(float), cudaMemcpyDeviceToHost));
  if (pi_out) CK(cudaMemcpy(pi_out, h->pi_out, B * A * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

int b2g_set_norm_stats(b2g_sac* h, const double* obs_mean, const double* obs_var, double ret_var, double clip_obs, double clip_rew,
                       double eps, int norm_obs, int norm_reward) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  if (norm_obs && !h->rms.on() && (!obs_mean || !obs_var)) return b2g_fail(B2G_EINVAL, "norm_obs needs obs_mean/obs_var");
  CK(cudaSetDevice(h->cfg.device));
  if (int rc = h->rms.norm_stats(obs_mean, obs_var, eps, h->cfg.device, h->cfg.nranks, h->allocs, h->stream)) return rc;
  if (h->rms.on()) obs_mean = obs_var = nullptr;
  // Called once per environment step by the learn loop (VecNormalize statistics move with every observation): the values
  // are staged in one of two pinned buffers and uploaded asynchronously IN STREAM ORDER -- no stream synchronisation, the
  // next gradient step simply sees them.  A buffer is reused only after its previous upload has completed.
  const int k = h->stats_k++ & 1;
  CK(cudaEventSynchronize(h->ev_stats[k]));
  double* st = h->hp_stats[k];
  const int Ec = h->Ec;
  if (norm_obs && obs_mean) {     // the caller's full-layout statistics, gathered into the ring layout
    double* m = st; double* is = st + Ec;
    for (int e = 0; e < Ec; ++e) {
      const int f = full_index(h, e);
      m[e] = f < 0 ? 0.0 : obs_mean[f];
      is[e] = f < 0 ? 1.0 : 1.0 / sqrt(obs_var[f] + eps);
    }
    CK(cudaMemcpyAsync(h->d_mean, m, Ec * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_istd, is, Ec * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    h->rms.up_other += (int64_t)(2 * h->E * sizeof(double));
  }
  h->ret_istd = 1.0 / sqrt(ret_var + eps);
  h->clip_obs = clip_obs; h->clip_rew = clip_rew; h->norm_obs = norm_obs; h->norm_rew = norm_reward;
  double* nc = st + 2 * Ec;
  nc[0] = h->ret_istd; nc[1] = clip_obs; nc[2] = clip_rew; nc[3] = (double)norm_obs; nc[4] = (double)norm_reward; nc[5] = nc[6] = nc[7] = 0.0;
  CK(cudaMemcpyAsync(h->d_normc, nc, 8 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  h->rms.up_other += 8 * sizeof(double);
  CK(cudaEventRecord(h->ev_stats[k], h->stream));
  return 0;
}

static int ensure_graph(b2g_sac* h) {
  if (h->graph_exec) return 0;
  int n = 0;
  if (int rc = capture_graph(h->stream, [&] { return issue_step(h, true, true, true, nullptr, &n); }, &h->graph_exec)) return rc;
  h->launches = n;
  return 0;
}

int b2g_sac_step_async(b2g_sac* h, int n_steps, float lr) {
  B2G_USABLE(h);
  if (!h || n_steps < 0) return b2g_fail(B2G_EINVAL, "bad argument");
  if (h->replay.size < 1) return b2g_fail(B2G_ESTATE, "replay buffer is empty");
  CK(cudaSetDevice(h->cfg.device));
  if (int rc = upload_lr(h->d_lr, &h->cur_lr, lr, h->stream)) return rc;
  refresh_planes(h, true);
  if (h->use_graph) if (int rc = ensure_graph(h)) return rc;
  CK(cudaEventRecord(h->ev0, h->stream));
  for (int i = 0; i < n_steps; ++i) {
    if (h->use_graph) CK(cudaGraphLaunch(h->graph_exec, h->stream));
    else if (int rc = issue_step(h, true, true, true, nullptr, &h->launches)) return rc;
  }
  CK(cudaEventRecord(h->ev1, h->stream));
  return 0;
}

int b2g_sac_step(b2g_sac* h, int n_steps, float lr, b2g_sac_metrics* out) {
  B2G_USABLE(h);
  if (int rc = b2g_sac_step_async(h, n_steps, lr)) return rc;
  if (int rc = fetch_metrics(h, out)) return rc;
  cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1);
  return 0;
}

int b2g_sac_step_explicit(b2g_sac* h, const float* obs, const float* act, const float* rew, const float* next_obs, const float* done,
                          const float* eps, float lr, int apply_update, b2g_sac_metrics* out, float* per_sample, float* pi_out) {
  B2G_USABLE(h);
  if (!h || !obs || !act || !rew || !next_obs || !done || !eps) return b2g_fail(B2G_EINVAL, "NULL argument");
  CK(cudaSetDevice(h->cfg.device));
  if (int rc = upload_lr(h->d_lr, &h->cur_lr, lr, h->stream)) return rc;
  const size_t B = h->B, A = h->A;
  refresh_planes(h, true);
  CK(cudaEventRecord(h->ev0, h->stream));
  if (int rc = load_rows(h, obs, h->s_obs, 0, B, B)) return rc;
  if (int rc = load_rows(h, next_obs, h->s_next, 0, B, B)) return rc;
  CK(cudaMemcpyAsync(h->s_act, act, B * A * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaMemcpyAsync(h->s_rew, rew, B * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaMemcpyAsync(h->s_done, done, B * sizeof(float), cudaMemcpyDefault, h->stream));
  CK(cudaMemcpyAsync(h->eps, eps, B * A * sizeof(float), cudaMemcpyDefault, h->stream));
  int n = 0;
  if (int rc = issue_step(h, false, apply_update != 0, true, nullptr, &n)) return rc;
  CK(cudaEventRecord(h->ev1, h->stream));
  if (per_sample) CK(cudaMemcpyAsync(per_sample, h->per_sample, 7 * B * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  if (pi_out) CK(cudaMemcpyAsync(pi_out, h->pi_out, B * A * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  if (int rc = fetch_metrics(h, out)) return rc;
  cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1);
  return 0;
}

namespace {
// full observations [n][HW][Cfull] -> compact replay rows [n][Ec] = image planes | value of the actuator plane at pixel [0,0] | pad
// (same layout compact_kernel writes on the device).  The actuator plane is constant over the image and the network only ever reads
// its first pixel (custom_obs_policy.py:20-23), so half of a depth observation never has to cross PCIe.
void compact_host(const float* src, float* dst, int n, int HW, int Cfull, int Ec, int threads) {
  const int Ci = Cfull - 1;
#pragma omp parallel for num_threads(threads) schedule(static)
  for (int b = 0; b < n; ++b) {
    const float* s = src + (size_t)b * HW * Cfull;
    float* d = dst + (size_t)b * Ec;
    if (Ci == 1) {
      for (int p = 0; p < HW; ++p) d[p] = s[2 * p];
    } else {
      for (int p = 0; p < HW; ++p)
        for (int c = 0; c < Ci; ++c) d[p * Ci + c] = s[p * Cfull + c];
    }
    d[HW * Ci] = s[Ci]; d[HW * Ci + 1] = 0.f; d[HW * Ci + 2] = 0.f; d[HW * Ci + 3] = 0.f;
  }
}

// the plain nature_cnn's compact rows: the whole observation [HW][C], then 4 zero floats
void copy_rows_host(const float* src, float* dst, int n, int E, int Ec, int threads) {
#pragma omp parallel for num_threads(threads) schedule(static)
  for (int b = 0; b < n; ++b) {
    float* d = dst + (size_t)b * Ec;
    memcpy(d, src + (size_t)b * E, (size_t)E * sizeof(float));
    d[E] = d[E + 1] = d[E + 2] = d[E + 3] = 0.f;
  }
}

void rows_host(const b2g_sac* h, const float* src, float* dst) {
  if (h->direct_feature()) compact_host(src, dst, h->B, h->Hi * h->Wi, h->Cobs, h->Ec, h->host_threads);
  else copy_rows_host(src, dst, h->B, h->E, h->Ec, h->host_threads);
}
}  // namespace

int b2g_debug_compact_host(const float* src, float* dst, int n, int hw, int cfull, int threads) {
  /* host-only (no device needed): the row compaction b2g_sac_step_host_pipelined applies before its copy */
  if (!src || !dst || n < 0 || hw < 1 || cfull < 2) return b2g_fail(B2G_EINVAL, "b2g_debug_compact_host: bad argument");
  compact_host(src, dst, n, hw, cfull, hw * (cfull - 1) + 4, threads > 0 ? threads : 1);
  return 0;
}

int b2g_sac_step_host_pipelined(b2g_sac* h, const float* obs, const float* act, const float* rew, const float* next_obs,
                                const float* done, const float* eps, float lr, b2g_sac_metrics* prev_out, int* have_prev) {
  B2G_USABLE(h);
  if (!h || !obs || !act || !rew || !next_obs || !done || !eps) return b2g_fail(B2G_EINVAL, "NULL argument");
  CK(cudaSetDevice(h->cfg.device));
  if (int rc = upload_lr(h->d_lr, &h->cur_lr, lr, h->stream)) return rc;
  refresh_planes(h, true);
  const size_t B = h->B, E = h->E, A = h->A;
  const long long k = h->pipe_k++;
  const int j = (int)(k & 1);
  // bring-up: B2G_PIPE_TRACE=1 prints, per call, when the copies and the kernels of the step two calls back ran on the device
  static const bool ptrace = getenv("B2G_PIPE_TRACE") != nullptr;
  static cudaEvent_t te[2][4], t_origin;
  static bool te_init = false;
  if (ptrace && !te_init) {
    for (auto& r : te) for (auto& e : r) cudaEventCreate(&e);
    cudaEventCreate(&t_origin); cudaEventRecord(t_origin, h->stream);
    te_init = true;
  }
  if (ptrace && k >= 2) {
    float c0, c1, k0, k1;
    cudaEventSynchronize(te[j][3]);
    cudaEventElapsedTime(&c0, t_origin, te[j][0]); cudaEventElapsedTime(&c1, t_origin, te[j][1]);
    cudaEventElapsedTime(&k0, t_origin, te[j][2]); cudaEventElapsedTime(&k1, t_origin, te[j][3]);
    fprintf(stderr, "pipe step %lld: copies %.3f .. %.3f ms (%.3f), kernels %.3f .. %.3f ms (%.3f)\n", k - 2, c0, c1, c1 - c0, k0, k1, k1 - k0);
  }
  // (1) copy stream: this step's observations into staging slot j (free once the gather of step k-2 has run)
  // staging slot j is free once step k-2 has run (its losses' event: the step replays as a graph, so no event from inside it)
  if (k >= 2) CK(cudaStreamWaitEvent(h->cstream, h->use_graph ? h->ev_met[j] : h->ev_consumed[j], 0));
  // Copy k+1 may or may not overlap the kernels of step k: on some machines the host-to-device copy and the step run side by side
  // at full speed, on others they starve each other and back to back wins.  So the first calls time both schedules (eight calls each, host clock, pipeline full) and the
  // faster one stays.  B2G_PIPE_MODE=overlap|serial pins it.  Either way the HOST stays pipelined: a call returns while its
  // copies and kernels are still queued.
  {
    static const char* pm = getenv("B2G_PIPE_MODE");
    const double now = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
    if (pm && pm[0] == 'o') h->pipe_serial = false;
    else if (pm && pm[0] == 's') h->pipe_serial = true;
    else if (h->pipe_tune < 22) {
      const int c = h->pipe_tune++;
      if (c == 4 || c == 14) h->pipe_t0 = now;
      if (c == 12) { h->pipe_period[0] = (now - h->pipe_t0) / 8; h->pipe_serial = true; }
      if (c == 21) {
        h->pipe_period[1] = (now - h->pipe_t0) / 7; h->pipe_serial = h->pipe_period[1] < h->pipe_period[0];
        if (getenv("B2G_PIPE_TRACE")) fprintf(stderr, "pipe schedule: overlapped %.3f ms/step, back to back %.3f ms/step -> %s\n", h->pipe_period[0] * 1e3, h->pipe_period[1] * 1e3, h->pipe_serial ? "back to back" : "overlapped");
      }
    }
  }
  if (h->pipe_serial && k >= 1) CK(cudaStreamWaitEvent(h->cstream, h->ev_met[j ^ 1], 0));
  if (ptrace) cudaEventRecord(te[j][0], h->cstream);
  if (h->cnn) {
    // compact on the host (a few threads, ~0.1 ms) into pinned staging, copy half the bytes; the caller's arrays need not be
    // pinned and are free again when this call returns
    if (!h->hc_obs[0]) {
      for (int q = 0; q < 2; ++q) {
        CK(cudaHostAlloc((void**)&h->hc_obs[q], B * h->Ec * sizeof(float), cudaHostAllocDefault));
        CK(cudaHostAlloc((void**)&h->hc_next[q], B * h->Ec * sizeof(float), cudaHostAllocDefault));
      }
      if (const char* e = getenv("B2G_HOST_THREADS")) h->host_threads = std::max(1, atoi(e));
    }
    if (k >= 2) CK(cudaEventSynchronize(h->ev_h2d[j]));          // the copy out of this staging slot two calls ago
    rows_host(h, obs, h->hc_obs[j]);
    CK(cudaMemcpyAsync(h->ps_obs[j], h->hc_obs[j], B * h->Ec * sizeof(float), cudaMemcpyHostToDevice, h->cstream));     // flies while next_obs is compacted
    rows_host(h, next_obs, h->hc_next[j]);
    CK(cudaMemcpyAsync(h->ps_next[j], h->hc_next[j], B * h->Ec * sizeof(float), cudaMemcpyHostToDevice, h->cstream));
  } else {
    CK(cudaMemcpyAsync(h->ps_obs[j], obs, B * E * sizeof(float), cudaMemcpyHostToDevice, h->cstream));
    CK(cudaMemcpyAsync(h->ps_next[j], next_obs, B * E * sizeof(float), cudaMemcpyHostToDevice, h->cstream));
  }
  CK(cudaEventRecord(h->ev_h2d[j], h->cstream));
  if (ptrace) cudaEventRecord(te[j][1], h->cstream);
  // (2) compute stream: small tensors in order, then the step on slot j
  CK(cudaMemcpyAsync(h->s_act, act, B * A * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(h->s_rew, rew, B * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(h->s_done, done, B * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(h->eps, eps, B * A * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamWaitEvent(h->stream, h->ev_h2d[j], 0));
  if (ptrace) cudaEventRecord(te[j][2], h->stream);
  float* keep_obs = h->s_obs; float* keep_next = h->s_next;
  h->s_obs = h->ps_obs[j]; h->s_next = h->ps_next[j];
  int n = 0, rc = 0;
  if (h->use_graph) {
    // one graph per staging slot (the slot's buffers are baked into the nodes): the ~30 runtime calls of an eagerly issued step
    // were the bottleneck of this path once the copy had shrunk
    if (!h->pipe_graph[j]) rc = capture_graph(h->stream, [&] { return issue_step(h, false, true, false, nullptr, &n); }, &h->pipe_graph[j]);
    if (!rc && cudaGraphLaunch(h->pipe_graph[j], h->stream) != cudaSuccess) rc = b2g_fail(B2G_ECUDA, "graph launch failed");
  } else {
    h->record_after_gather = h->ev_consumed[j];
    rc = issue_step(h, false, true, false, nullptr, &n);
    h->record_after_gather = nullptr;
  }
  h->s_obs = keep_obs; h->s_next = keep_next;
  if (rc) return rc;
  if (ptrace) cudaEventRecord(te[j][3], h->stream);
  // (3) this step's losses -> pinned slot j (read back by the NEXT call, or by b2g_sac_pipeline_flush)
  if (int rc = copy_metrics_async(h, h->pm_met[j], h->pm_cnt[j])) return rc;
  CK(cudaEventRecord(h->ev_met[j], h->stream));
  // (4) hand back the PREVIOUS step's losses: blocks only until step k-1 has finished, while step k's copies run
  if (have_prev) *have_prev = h->pipe_pending ? 1 : 0;
  if (h->pipe_pending) {
    CK(cudaEventSynchronize(h->ev_met[j ^ 1]));
    if (prev_out) fill_metrics(h, h->pm_met[j ^ 1], h->pm_cnt[j ^ 1], prev_out);
  }
  h->pipe_pending = true;
  return 0;
}

int b2g_sac_pipeline_flush(b2g_sac* h, b2g_sac_metrics* last_out) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  CK(cudaSetDevice(h->cfg.device));
  if (!h->pipe_pending) return b2g_fail(B2G_ESTATE, "no pipelined step in flight");
  const int j = (int)((h->pipe_k - 1) & 1);
  CK(cudaEventSynchronize(h->ev_met[j]));
  if (last_out) fill_metrics(h, h->pm_met[j], h->pm_cnt[j], last_out);
  h->pipe_pending = false;
  return 0;
}

int b2g_sac_act(b2g_sac* h, const float* obs, int n, int deterministic, float* act_out) {
  B2G_USABLE(h);
  if (!h || !obs || !act_out || n < 0) return b2g_fail(B2G_EINVAL, "bad argument");
  CK(cudaSetDevice(h->cfg.device));
  const size_t E = h->E, A = h->A;
  for (int done_n = 0; done_n < n; done_n += h->B) {
    const int chunk = std::min(h->B, n - done_n);
    if (int rc = load_rows(h, obs + (size_t)done_n * E, h->s_obs, 0, h->B, chunk)) return rc;
    h->rms.up_other += (int64_t)(chunk * E * sizeof(float));
    if (int rc = sac_act_rows(h, h->s_obs, chunk, deterministic)) return rc;
    CK(cudaMemcpyAsync(act_out + (size_t)done_n * A, h->pi_out, chunk * A * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  CK(cudaGetLastError());
  return 0;
}

int b2g_launches_per_step(const b2g_sac* h) {
  B2G_USABLE(h);
  if (!h) return 0;
  if (h->launches) return h->launches;
  // prep + gather + memset + groups + tail + optim (+3 with a collective)
  return 3 + (int)h->fwd_groups.size() + 1 + (int)h->bwd_groups.size() + 1 + (h->cfg.nranks > 1 ? 3 : 0);
}

float b2g_last_step_ms(const b2g_sac* h) { B2G_USABLE(h); return h ? h->last_ms : 0.f; }

int b2g_profile_step(b2g_sac* h, float lr, const char** names, float* ms, int cap) {
  B2G_USABLE(h);
  if (!h || !names || !ms) return b2g_fail(B2G_EINVAL, "NULL argument");
  if (h->replay.size < 1) return b2g_fail(B2G_ESTATE, "replay buffer is empty");
  CK(cudaSetDevice(h->cfg.device));
  if (int rc = upload_lr(h->d_lr, &h->cur_lr, lr, h->stream)) return rc;
  refresh_planes(h);
  Prof prof;
  prof.on = true;
  int n = 0;
  if (int rc = issue_step(h, true, true, false, &prof, &n)) return rc;
  CK(cudaStreamSynchronize(h->stream));
  h->prof_names = prof.names;
  int k = 0;
  for (size_t i = 1; i < prof.ev.size() && k < cap; ++i, ++k) {
    cudaEventElapsedTime(&ms[k], prof.ev[i - 1], prof.ev[i]);
    names[k] = h->prof_names[i].c_str();
  }
  for (auto e : prof.ev) cudaEventDestroy(e);
  return k;
}

}  // extern "C"

// ================================================================================================
// Training state (b2g_sac_state_save / _load; container format in state.cuh)
// ================================================================================================
namespace {

std::vector<FpField> sac_fingerprint(const b2g_sac* h) {
  const b2g_sac_cfg& c = h->cfg;
  return {fp_int("obs_h", c.obs_h), fp_int("obs_w", c.obs_w), fp_int("obs_c", c.obs_c), fp_int("obs_dim", c.obs_dim),
          fp_int("n_act", c.n_act), fp_int("hidden", c.hidden), fp_int("batch", c.batch),
          fp_int("buffer_capacity", c.buffer_capacity), fp_int("frame_capacity", h->replay.ring.frame_cap),
          fp_int("u8_plane_mask", h->u8_mask), fp_real("gamma", c.gamma), fp_real("tau", c.tau),
          fp_real("target_entropy", c.target_entropy), fp_int("seed", (int64_t)c.seed)};
}

// the augmented and MLP fingerprints carry no extractor field, so their files keep the layout they had before nature_cnn existed
std::vector<FpField> sac_fingerprint(const b2g_sac* h, int extractor) {
  std::vector<FpField> fp = sac_fingerprint(h);
  if (extractor == B2G_CNN_NATURE) fp.push_back(fp_int("extractor", extractor));
  return fp;
}

// the sections 2.. (parameters .. frames, then obs_rms when the handle owns it) of a handle whose frame window is [lo, hi)
std::vector<StateSection> sac_device_sections(b2g_sac* h, int64_t lo, int64_t hi) {
  std::vector<StateSection> s = adam_sections(h->P, h->n_all, h->Mo, h->Vo, h->n_train);
  for (auto& r : h->replay.state_sections(0, lo, hi)) s.push_back(std::move(r));     // ROFR RNFR RACT RREW RDON FRMS
  if (h->rms.on()) s.push_back(rms_section(&h->rms.count, h->rms.mean, h->rms.var, h->E));
  return s;
}

}  // namespace

extern "C" {

int b2g_sac_state_save(b2g_sac* h, const char* path) {
  if (!h || !path) return b2g_fail(B2G_EINVAL, "NULL argument");
  B2G_USABLE(h);
  if (h->cfg.nranks > 1)
    return b2g_fail(B2G_ESTATE, "training-state files of data-parallel learners (nranks > 1) are not built: each rank holds only its "
                                "slice of the Adam moments");
  if (h->pipe_pending)
    return b2g_fail(B2G_ESTATE, "a host-pipelined step is in flight: call b2g_sac_pipeline_flush first (its losses would be lost)");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));     // every enqueued step (b2g_sac_step_async included) has run
  if (h->aux) { CK(cudaStreamSynchronize(h->aux)); CK(cudaStreamSynchronize(h->aux2)); }
  long long cnt[8];
  CK(cudaMemcpy(cnt, h->counters, sizeof cnt, cudaMemcpyDeviceToHost));
  const FrameRing& ring = h->replay.ring;
  std::vector<int64_t> hv = ring.pack();     // the replay's bookkeeping (its size is replay.size)
  std::vector<StateSection> secs = host_sections(hv.data(), hv.size() * sizeof(int64_t), cnt, sizeof cnt);
  for (auto& s : sac_device_sections(h, ring.frame_lo(), ring.next_fid)) secs.push_back(std::move(s));
  return state_write(path, STATE_KIND_SAC, fp_with_rms(sac_fingerprint(h, h->extractor), h->rms.on()), secs);
}

int b2g_sac_state_load(b2g_sac* h, const char* path) {
  if (!h || !path) return b2g_fail(B2G_EINVAL, "NULL argument");
  if (h->cfg.nranks > 1)
    return b2g_fail(B2G_ESTATE, "training-state files of data-parallel learners (nranks > 1) are not built");
  if (h->pipe_pending)
    return b2g_fail(B2G_ESTATE, "a host-pipelined step is in flight: call b2g_sac_pipeline_flush first");
  CK(cudaSetDevice(h->cfg.device));
  // ---- everything is checked before the handle changes
  StateReader rd;
  if (int rc = state_open_rms(rd, path, STATE_KIND_SAC, sac_fingerprint(h, h->extractor), h->rms.on(), h->rms.set_call)) {
    const std::string msg = g_b2g_err;
    StateReader other;      // a file of the other CNN extractor: say so
    const int ext2 = h->extractor == B2G_CNN_NATURE ? B2G_CNN_AUGMENTED : B2G_CNN_NATURE;
    if (h->cnn && other.open(path, STATE_KIND_SAC, fp_with_rms(sac_fingerprint(h, ext2), h->rms.on())) == 0)
      return b2g_fail(B2G_EINVAL, std::string("the state file was written by a handle of the ") +
                                      (ext2 == B2G_CNN_NATURE ? "nature_cnn" : "augmented") + " extractor; this handle runs the " +
                                      (ext2 == B2G_CNN_NATURE ? "augmented" : "nature_cnn") + " one");
    return b2g_fail(rc, msg);
  }
  if (int rc = state_check_tags(rd, sac_device_sections(h, 0, 0), "SAC")) return rc;
  const int64_t cap = h->cfg.buffer_capacity, FC = h->replay.ring.frame_cap;
  if (rd.bytes(0) % 8 || rd.bytes(0) < 7 * 8 || rd.bytes(0) > (uint64_t)(7 + 2 * cap + 4 * FC) * 8)
    return b2g_fail(B2G_EINVAL, "corrupt replay bookkeeping in the training-state file");
  std::vector<int64_t> hv(rd.bytes(0) / 8);
  if (int rc = rd.read_host(0, hv.data(), hv.size() * 8)) return rc;
  FrameRing hs = h->replay.ring;
  if (!hs.unpack(hv.data(), hv.size(), cap)) return b2g_fail(B2G_EINVAL, "corrupt replay bookkeeping in the training-state file");
  const std::vector<StateSection> dev = sac_device_sections(h, hs.frame_lo(), hs.next_fid);
  if (int rc = state_check_lengths(rd, dev)) return rc;
  long long cnt[8];
  if (rd.bytes(1) != sizeof cnt) return b2g_fail(B2G_EINVAL, "training-state section lengths do not match this handle's configuration");
  if (int rc = rd.read_host(1, cnt, sizeof cnt)) return rc;
  // ---- from here on a failure leaves the handle unusable until a load succeeds
  CK(cudaStreamSynchronize(h->stream));
  if (h->aux) { CK(cudaStreamSynchronize(h->aux)); CK(cudaStreamSynchronize(h->aux2)); }
  return state_read_device(rd, dev, &h->broken, [&] {
    if (h->rms.on()) h->rms.derive(h->stream);
    h->ob_n = 0;       // staged observations name frames of the replaced replay: the next b2g_sac_observe_act stages anew
    CK(cudaMemcpy(h->counters, cnt, sizeof cnt, cudaMemcpyHostToDevice));
    h->replay.ring = hs;
    h->replay.size = hs.size();
    h->replay.pos = hs.head_seq % cap;
    // The BF16 weight planes follow the restored arena at the next step or act.  The captured step graphs (graph_exec, pipe_graph)
    // stay valid: their kernel parameters hold device pointers and configuration only, and the replay size, first live slot and
    // Philox step they depend on are read from the device counters restored above.
    h->planes_dirty = true;
    return mlog_rebase(&h->mlog, h->counters + 3, h->stream);     // the restored counter: rows before it are not pending
  });
}

int b2g_sac_metrics_log(b2g_sac* h, int capacity) {
  B2G_USABLE(h);
  if (!h || capacity < 0) return b2g_fail(B2G_EINVAL, "bad argument");
  if (h->pipe_pending) return b2g_fail(B2G_ESTATE, "a host-pipelined step is in flight: call b2g_sac_pipeline_flush first");
  CK(cudaSetDevice(h->cfg.device));
  if (h->aux) { CK(cudaStreamSynchronize(h->aux)); CK(cudaStreamSynchronize(h->aux2)); }
  if (int rc = mlog_enable(&h->mlog, capacity, B2G_SAC_LOG_COLS, h->counters + 3, h->stream)) return rc;
  // the step gains or loses its append node: capture again at the next step
  if (h->graph_exec) { cudaGraphExecDestroy(h->graph_exec); h->graph_exec = nullptr; }
  for (auto& g : h->pipe_graph) if (g) { cudaGraphExecDestroy(g); g = nullptr; }
  h->launches = 0;
  return 0;
}

int b2g_sac_metrics_drain(b2g_sac* h, float* rows, int max_rows, int64_t* first_step, int* n_rows, int64_t* lost) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL handle");
  CK(cudaSetDevice(h->cfg.device));
  const float inv = 1.0f / (float)h->cfg.nranks;
  return mlog_drain(&h->mlog, h->counters + 3, h->stream, rows, max_rows, first_step, n_rows, lost, [inv](float* r) {
    for (int k = 0; k < 6; ++k) r[k] *= inv;     // as fill_metrics
    r[6] = expf(r[6]);
  });
}

}  // extern "C"
