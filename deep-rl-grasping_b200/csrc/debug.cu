// Bring-up / measurement hooks of libb200grasp (not on the product path).
//
// b2g_debug_gemm: one dense C[M,N] = A[M,K] * B[N,K]^T through the wgmma gather-GEMM engine (register-staged fp32
// operands, BF16 hi/lo split when x3 != 0), used by tools/tc_accum_probe.py to measure what the tensor core's fp32
// accumulation in registers does to long, cancelling reductions -- independently of the operand split.
// b2g_debug_tensor_info / b2g_debug_tensor: one plane of one named device tensor of a SAC handle (engine v2 planes, fp32 head
// buffers) back to the host, so that tests can hold each contraction to a float64 contraction of the inputs it actually read.
#include <cuda_runtime.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "../../include/b200grasp.h"
#include "common.cuh"
#include "sac_internal.cuh"

using namespace b2g;

namespace {
struct DebugTensor {
  const void* planes[3] = {nullptr, nullptr, nullptr};
  int np = 0, elem_bytes = 0;
  int64_t numel = 0;
  bool v2 = false;
};

// the layouts are documented with b2g_debug_tensor_info in b200grasp.h
int find_debug_tensor(const b2g_sac* h, const std::string& name, DebugTensor& t) {
  const V2State& v = h->v2;
  const int64_t B = h->B, H = h->H, KF = v.KF, Cp = s2d_channels(h->Cimg), K1 = 64 * Cp;
  const std::string net3[3] = {"pi", "values", "target"};
  const std::string head[4] = {"pi", "vf", "qf1", "qf2"};
  auto bf = [&](const uint16_t* const* p, int np, int64_t numel) {
    for (int k = 0; k < np; ++k) t.planes[k] = p[k];
    t.np = np; t.elem_bytes = 2; t.numel = numel; t.v2 = true;
    return 0;
  };
  auto f32 = [&](const float* p, int64_t numel) {
    t.planes[0] = p; t.np = 1; t.elem_bytes = 4; t.numel = numel; t.v2 = false;
    return 0;
  };
  if (name == "S/obs") return bf(v.S[0], 3, B * 4096 * Cp);
  if (name == "S/next_obs") return bf(v.S[1], 3, B * 4096 * Cp);
  if (name == "dz0pi") return bf(v.dz0pi, 2, B * H);
  if (name == "dz0v") return bf(v.dz0v, 2, B * 3 * H);
  if (name == "dZ1") return bf(v.dZ1, 2, B * 225 * 64);
  if (name == "W1T/online") return bf(v.W1T[0], 3, 64 * K1);
  if (name == "W1T/target") return bf(v.W1T[1], 3, 32 * K1);
  for (int n = 0; n < 3; ++n) {
    const std::string s = "/" + net3[n];
    if (name == "H1" + s) return bf(v.H1[n], 3, B * 225 * 32);
    if (name == "H2" + s) return bf(v.H2[n], 3, B * 36 * 64);
    if (name == "H3" + s) return bf(v.H3[n], 3, B * 1024);
    if (name == "F" + s) return bf(v.F[n], 3, B * KF);
    if (name == "W2T" + s) return bf(v.W2T[n], 3, 64 * 512);
    if (name == "W3T" + s) return bf(v.W3T[n], 3, 64 * 576);
    if (name == "WfT" + s) return bf(v.WfT[n], 3, 512 * 1024);
    if (name == "K0T" + s) return bf(v.K0T[n], 3, (n == 1 ? 3 : 1) * H * KF);
    if (name == "F32" + s) return f32(h->F[n], B * h->FS);
    if (n == 2) continue;
    if (name == "dZ4" + s) return bf(v.dZ4[n], 2, B * 512);
    if (name == "dZ3" + s) return bf(v.dZ3[n], 2, B * 1024);
    if (name == "dZ2" + s) return bf(v.dZ2[n], 2, B * 36 * 64);
    if (name == "W2n" + s) return bf(v.W2n[n], 2, 512 * 64);
    if (name == "W3n" + s) return bf(v.W3n[n], 2, 576 * 64);
    if (name == "Wfn" + s) return bf(v.Wfn[n], 2, 1024 * 512);
    if (name == "K0n" + s) return bf(v.K0n[n], 2, KF * (n == 1 ? 3 : 1) * H);
  }
  for (int q = 0; q < 4; ++q) {
    if (name == "a0/" + head[q]) return f32(h->a0[q], B * H);
    if (name == "dz1/" + head[q]) return f32(h->dz1[q], B * H);
  }
  if (name == "z0/pi") return f32(h->z0[0], B * H);
  if (name == "z0/target") return f32(h->z0[4], B * H);
  for (int q = 1; q < 4; ++q)      // separate buffers only without engine v2 (which writes them into z0v)
    if (name == "z0/" + head[q]) {
      if (v.on) return b2g_fail(B2G_ESTATE, name + ": engine v2 writes the value heads' fc0 outputs into z0v");
      return f32(h->z0[q], B * H);
    }
  if (name == "rew_n") return f32(h->rew_n, B);
  if (name == "done_n") return f32(h->done_n, B);
  if (name == "z0v") { t.v2 = true; t.planes[0] = v.z0v; t.np = 1; t.elem_bytes = 4; t.numel = B * 3 * H; return 0; }
  if (name == "dz0_pi") return f32(h->dz0_pi, B * H);
  if (name == "dz0_v3") return f32(h->dz0_v3, B * 3 * H);
  return b2g_fail(B2G_EINVAL, "unknown debug tensor: " + name);
}
}  // namespace

extern "C" int b2g_debug_tensor_info(const b2g_sac* h, const char* name, int64_t* numel, int32_t* planes, int32_t* elem_bytes) {
  B2G_USABLE(h);
  if (!h || !name) return b2g_fail(B2G_EINVAL, "NULL argument");
  DebugTensor t;
  if (int rc = find_debug_tensor(h, name, t)) return rc;
  if (t.v2 && !h->v2.on) return b2g_fail(B2G_ESTATE, std::string(name) + ": this handle does not run engine v2");
  if (!t.planes[0]) return b2g_fail(B2G_ESTATE, std::string(name) + ": not allocated on this handle");
  if (numel) *numel = t.numel;
  if (planes) *planes = t.np;
  if (elem_bytes) *elem_bytes = t.elem_bytes;
  return 0;
}

extern "C" int b2g_debug_tensor(b2g_sac* h, const char* name, int plane, void* dst, size_t bytes) {
  B2G_USABLE(h);
  if (!h || !name || !dst) return b2g_fail(B2G_EINVAL, "NULL argument");
  DebugTensor t;
  if (int rc = find_debug_tensor(h, name, t)) return rc;
  if (t.v2 && !h->v2.on) return b2g_fail(B2G_ESTATE, std::string(name) + ": this handle does not run engine v2");
  if (!t.planes[0]) return b2g_fail(B2G_ESTATE, std::string(name) + ": not allocated on this handle");
  if (plane < 0 || plane >= t.np) return b2g_fail(B2G_EINVAL, std::string(name) + ": plane out of range");
  if (bytes != (size_t)t.numel * t.elem_bytes) return b2g_fail(B2G_EINVAL, std::string(name) + ": size mismatch");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaMemcpy(dst, t.planes[plane], bytes, cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int b2g_debug_gemm(int M, int N, int K, const float* A, const float* B, float* C, int x3, int split_k) {
  if (M < 1 || N < 1 || K < 8 || (K & 7) || !A || !B || !C || split_k < 1) return B2G_EINVAL;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) return B2G_ECUDA;
  float *dA = nullptr, *dB = nullptr, *dC = nullptr;
  int* tabs = nullptr;
  std::vector<int> t((size_t)M + K + K + N + M + N);
  int* aM = t.data(); int* aR = aM + M; int* bR = aR + K; int* bN = bR + K; int* cM = bN + N; int* cN = cM + M;
  for (int m = 0; m < M; ++m) { aM[m] = m * K; cM[m] = m * N; }
  for (int r = 0; r < K; ++r) { aR[r] = r; bR[r] = r; }
  for (int n = 0; n < N; ++n) { bN[n] = n * K; cN[n] = n; }
  auto ck = [](cudaError_t e) { return e == cudaSuccess; };
  bool ok = ck(cudaMalloc(&dA, (size_t)M * K * 4)) && ck(cudaMalloc(&dB, (size_t)N * K * 4)) && ck(cudaMalloc(&dC, (size_t)M * N * 4)) &&
            ck(cudaMalloc(&tabs, t.size() * 4));
  ok = ok && ck(cudaMemcpy(dA, A, (size_t)M * K * 4, cudaMemcpyHostToDevice)) && ck(cudaMemcpy(dB, B, (size_t)N * K * 4, cudaMemcpyHostToDevice)) &&
       ck(cudaMemcpy(tabs, t.data(), t.size() * 4, cudaMemcpyHostToDevice)) && ck(cudaMemset(dC, 0, (size_t)M * N * 4));
  if (ok) {
    GemmDesc d{};
    d.A = dA; d.B = dB; d.C = dC;
    d.aM = tabs; d.aR = tabs + M; d.bR = tabs + M + K; d.bN = tabs + M + 2 * K; d.cM = tabs + M + 2 * K + N; d.cN = tabs + 2 * M + 2 * K + N;
    d.M = M; d.N = N; d.R = K;
    d.flags = GG_A_RVEC | GG_B_RVEC | (split_k > 1 ? GG_EPI_ATOMIC : 0);
    d.splitR = split_k;
    d.tiles_m = (M + GG_TC_BM - 1) / GG_TC_BM; d.tiles_n = (N + GG_TC_BN - 1) / GG_TC_BN;
    d.tile_start = 0; d.tile_count = d.tiles_m * d.tiles_n * d.splitR;
    cudaDeviceProp prop{};
    cudaGetDeviceProperties(&prop, 0);
    ok = ck(gg_tc_launch(&d, 1, d.tile_count, d.flags, x3 ? 1 : 0, prop.multiProcessorCount, 0)) && ck(cudaDeviceSynchronize()) &&
         ck(cudaMemcpy(C, dC, (size_t)M * N * 4, cudaMemcpyDeviceToHost));
  }
  cudaFree(dA); cudaFree(dB); cudaFree(dC); cudaFree(tabs);
  return ok ? 0 : B2G_ECUDA;
}

static_assert(B2G_GG_A_RVEC == GG_A_RVEC && B2G_GG_B_RVEC == GG_B_RVEC && B2G_GG_EPI_BIAS_RELU == GG_EPI_BIAS_RELU &&
                  B2G_GG_EPI_MASK == GG_EPI_MASK && B2G_GG_EPI_ATOMIC == GG_EPI_ATOMIC && B2G_GG_COLSUM == GG_COLSUM &&
                  B2G_GG_EPI_BIAS == GG_EPI_BIAS && B2G_GG_EPI_SCALE == GG_EPI_SCALE && B2G_GG_A_SCALAR == GG_A_SCALAR &&
                  B2G_GG_EPI_BIAS_LRELU == GG_EPI_BIAS_LRELU && B2G_GG_EPI_LRELU_GRAD == GG_EPI_LRELU_GRAD &&
                  B2G_GG_EPI_BIAS_TANH == GG_EPI_BIAS_TANH && B2G_GG_EPI_TANH_GRAD == GG_EPI_TANH_GRAD,
              "the public gg flag values follow common.cuh");

namespace {
// The contracts of gg_simt_body that hold only by construction at each call site, checked for one caller-described problem
// (the refusals are listed with b2g_debug_gg_simt in b200grasp.h).  0, or B2G_EINVAL with the broken contract named.
int check_gg_problem(int build, int idx, const b2g_debug_gg_problem& p, int64_t n_f32, int64_t n_f64, int64_t n_u16,
                     const int32_t* tabs, int64_t n_tabs) {
  const std::string at = "problem " + std::to_string(idx) + ": ";
  auto fail = [&](const std::string& why) { return b2g_fail(B2G_EINVAL, at + why); };
  const int f = p.flags;
  int allowed = GG_A_RVEC | GG_B_RVEC | GG_EPI_BIAS_RELU | GG_EPI_MASK | GG_EPI_ATOMIC | GG_COLSUM | GG_EPI_BIAS | GG_EPI_SCALE |
                GG_A_SCALAR | GG_EPI_BIAS_LRELU;
  if (build == 1) allowed |= GG_EPI_LRELU_GRAD;
  if (build == 2) allowed |= GG_EPI_BIAS_TANH | GG_EPI_TANH_GRAD;
  if (f & ~allowed) return fail("flags " + std::to_string(f & ~allowed) + " are not flags of build " + std::to_string(build));
  if ((f & GG_A_SCALAR) && !(f & GG_A_RVEC) && build != 1) return fail("m-direction GG_A_SCALAR exists in build 1 only");
  if (p.M < 1 || p.N < 1 || p.R < 1) return fail("M, N and R must be >= 1");
  if (p.splitR < 1 || p.splitR > p.R) return fail("splitR must be in 1..R");
  if (p.splitR > 1 && !(f & GG_EPI_ATOMIC)) return fail("splitR > 1 needs GG_EPI_ATOMIC (the splits would overwrite each other)");
  if ((f & GG_COLSUM) && (f & GG_B_RVEC)) return fail("GG_COLSUM sums the n-direction B loads; it cannot take GG_B_RVEC");
  const bool c64 = build == 1 && (f & GG_EPI_ATOMIC), s64 = build == 1 && (f & GG_COLSUM);
  const bool need_bias = f & (GG_EPI_BIAS_RELU | GG_EPI_BIAS | GG_EPI_BIAS_LRELU | GG_EPI_BIAS_TANH);
  const bool need_mask = f & (GG_EPI_MASK | GG_EPI_LRELU_GRAD | GG_EPI_TANH_GRAD);
  if (p.A < 0 || p.B < 0 || p.C < 0) return fail("A, B and C are required");
  if (need_bias != (p.bias >= 0)) return fail(need_bias ? "the bias epilogue needs bias" : "bias given without a bias epilogue");
  if (need_mask != (p.mask >= 0)) return fail(need_mask ? "the mask epilogue needs mask" : "mask given without a mask epilogue");
  if (((f & GG_COLSUM) != 0) != (p.colsum >= 0)) return fail("colsum goes with GG_COLSUM");
  if ((p.C_hi >= 0) != (p.C_lo >= 0)) return fail("C_hi and C_lo go together");
  if ((f & GG_EPI_ATOMIC) && p.C_hi >= 0) return fail("C_hi / C_lo would hold one split's partial under GG_EPI_ATOMIC");
  if (p.C % 4) return fail("C must be 16-byte aligned (the float4 output store)");
  // tables
  struct Tab { const char* name; int64_t off; int len; const int32_t* v = nullptr; int64_t lo = 0, hi = 0; };
  Tab t[8] = {{"aM", p.aM, p.M}, {"aR", p.aR, p.R}, {"bR", p.bR, p.R}, {"bN", p.bN, p.N},
              {"cM", p.cM, p.M}, {"cN", p.cN, p.N}, {"kM", p.kM, p.M}, {"kN", p.kN, p.N}};
  for (int i = 0; i < 8; ++i) {
    if (t[i].off < 0) {
      if (i < 6) return fail(std::string(t[i].name) + " is required");
      t[i] = t[i - 2];          // kM / kN default to cM / cN
      continue;
    }
    if (t[i].off + t[i].len > n_tabs) return fail(std::string(t[i].name) + " runs past the end of tabs");
    t[i].v = tabs + t[i].off;
    t[i].lo = *std::min_element(t[i].v, t[i].v + t[i].len);
    t[i].hi = *std::max_element(t[i].v, t[i].v + t[i].len);
  }
  const Tab &aM = t[0], &aR = t[1], &bR = t[2], &bN = t[3], &cM = t[4], &cN = t[5], &kM = t[6], &kN = t[7];
  auto in = [&](const char* what, int64_t base, int64_t lo, int64_t hi, int64_t n) {
    return base + lo >= 0 && base + hi < n ? 0 : fail(std::string(what) + " reaches outside its arena");
  };
  if (int rc = in("A[aM + aR]", p.A, aM.lo + aR.lo, aM.hi + aR.hi, n_f32)) return rc;
  if (int rc = in("B[bR + bN]", p.B, bR.lo + bN.lo, bR.hi + bN.hi, n_f32)) return rc;
  if (int rc = in("C[cM + cN]", p.C, cM.lo + cN.lo, cM.hi + cN.hi, c64 ? n_f64 : n_f32)) return rc;
  if (p.C_hi >= 0) {
    if (int rc = in("C_hi[cM + cN]", p.C_hi, cM.lo + cN.lo, cM.hi + cN.hi, n_u16)) return rc;
    if (int rc = in("C_lo[cM + cN]", p.C_lo, cM.lo + cN.lo, cM.hi + cN.hi, n_u16)) return rc;
  }
  if (need_bias) if (int rc = in("bias[n]", p.bias, 0, p.N - 1, n_f32)) return rc;
  if (need_mask) if (int rc = in("mask[kM + kN]", p.mask, kM.lo + kN.lo, kM.hi + kN.hi, n_f32)) return rc;
  if (f & GG_COLSUM) if (int rc = in("colsum[n]", p.colsum, 0, p.N - 1, s64 ? n_f64 : n_f32)) return rc;
  // 4-groups: r-vector loads take r in [4g, 4g + 4) when 4g + 3 < R (splits start at multiples of 16); m- / n-direction loads
  // take rows (columns) [4g, 4g + 4) when 4g + 3 < M (N).  Each taken group must be contiguous, and base + the group's first
  // offset + every offset of the other side 16-byte aligned.
  auto groups = [&](const char* what, int64_t base, const Tab& g, const Tab& other) {
    for (int i = 0; i + 3 < g.len; i += 4)
      for (int j = 1; j < 4; ++j)
        if (g.v[i + j] != g.v[i] + j) return fail(std::string(what) + ": " + g.name + " is not contiguous in the 4-group at " + std::to_string(i));
    if (g.len < 4) return 0;
    for (int i = 0; i + 3 < g.len; i += 4)
      if ((base + g.v[i] + other.v[0]) & 3) return fail(std::string(what) + ": the 4-groups of " + g.name + " are not 16-byte aligned");
    for (int i = 0; i < other.len; ++i)
      if ((base + g.v[0] + other.v[i]) & 3) return fail(std::string(what) + ": the 4-groups of " + g.name + " are not 16-byte aligned");
    return 0;
  };
  if (f & GG_A_RVEC) {
    if (!(f & GG_A_SCALAR)) if (int rc = groups("GG_A_RVEC", p.A, aR, aM)) return rc;
  } else if (!(build == 1 && (f & GG_A_SCALAR))) {
    if (int rc = groups("m-direction A", p.A, aM, aR)) return rc;
  }
  if (f & GG_B_RVEC) {
    if (int rc = groups("GG_B_RVEC", p.B, bR, bN)) return rc;
  } else if (int rc = groups("n-direction B", p.B, bN, bR)) return rc;
  return 0;
}
}  // namespace

extern "C" int b2g_debug_gg_simt(int build, const b2g_debug_gg_problem* p, int n, float* f32, int64_t n_f32, double* f64, int64_t n_f64,
                                 uint16_t* u16, int64_t n_u16, const int32_t* tabs, int64_t n_tabs) {
  if (build < 0 || build > 2) return b2g_fail(B2G_EINVAL, "build must be 0 (plain), 1 (ext) or 2 (tanh)");
  if (!p || n < 1 || n > 16) return b2g_fail(B2G_EINVAL, "1 to 16 problems per launch");
  const int64_t lim = (int64_t)1 << 31;
  if (n_f32 < 0 || n_f64 < 0 || n_u16 < 0 || n_tabs < 0 || n_f32 >= lim || n_f64 >= lim || n_u16 >= lim || n_tabs >= lim)
    return b2g_fail(B2G_EINVAL, "arena lengths must be in 0 .. 2^31 - 1");
  if ((n_f32 && !f32) || (n_f64 && !f64) || (n_u16 && !u16) || (n_tabs && !tabs)) return b2g_fail(B2G_EINVAL, "NULL arena");
  for (int i = 0; i < n; ++i)
    if (int rc = check_gg_problem(build, i, p[i], n_f32, n_f64, n_u16, tabs, n_tabs)) return rc;

  if (int rc = check_device(0)) return rc;
  cudaStream_t s = nullptr;
  CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  std::vector<void*> allocs;
  const int rc = [&]() -> int {
    float* d32 = nullptr; double* d64 = nullptr; uint16_t* d16 = nullptr; int32_t* dt = nullptr;
    if (int rc = dev_alloc(allocs, s, &d32, n_f32, false)) return rc;
    if (int rc = dev_alloc(allocs, s, &d64, n_f64, false)) return rc;
    if (int rc = dev_alloc(allocs, s, &d16, n_u16, false)) return rc;
    if (int rc = dev_alloc(allocs, s, &dt, n_tabs, false)) return rc;
    if (n_f32) CK(cudaMemcpyAsync(d32, f32, n_f32 * sizeof(float), cudaMemcpyHostToDevice, s));
    if (n_f64) CK(cudaMemcpyAsync(d64, f64, n_f64 * sizeof(double), cudaMemcpyHostToDevice, s));
    if (n_u16) CK(cudaMemcpyAsync(d16, u16, n_u16 * sizeof(uint16_t), cudaMemcpyHostToDevice, s));
    if (n_tabs) CK(cudaMemcpyAsync(dt, tabs, n_tabs * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    GemmGroup g;
    g.name = "debug_gg_simt";
    for (int i = 0; i < n; ++i) {
      const b2g_debug_gg_problem& q = p[i];
      const bool c64 = build == 1 && (q.flags & GG_EPI_ATOMIC), s64 = build == 1 && (q.flags & GG_COLSUM);
      GemmDesc d = gemm_desc(d32 + q.A, dt + q.aM, dt + q.aR, d32 + q.B, dt + q.bR, dt + q.bN,
                             c64 ? reinterpret_cast<float*>(d64 + q.C) : d32 + q.C, dt + q.cM, dt + q.cN, q.M, q.N, q.R, q.flags, q.splitR);
      if (q.kM >= 0) d.kM = dt + q.kM;
      if (q.kN >= 0) d.kN = dt + q.kN;
      if (q.bias >= 0) d.bias = d32 + q.bias;
      if (q.mask >= 0) d.mask = d32 + q.mask;
      if (q.colsum >= 0) d.colsum = s64 ? reinterpret_cast<float*>(d64 + q.colsum) : d32 + q.colsum;
      if (q.C_hi >= 0) { d.C_hi = d16 + q.C_hi; d.C_lo = d16 + q.C_lo; }
      d.alpha = q.alpha;
      g.host.push_back(d);
    }
    if (int rc = finalize_tiles(g, allocs, s)) return rc;
    if (build == 0) gg_simt_launch(g.dev, n, g.total_tiles, s);
    else if (build == 1) gg_simt_launch_ext(g.dev, n, g.total_tiles, s);
    else gg_simt_launch_tanh(g.dev, n, g.total_tiles, s);
    CK(cudaGetLastError());
    if (n_f32) CK(cudaMemcpyAsync(f32, d32, n_f32 * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (n_f64) CK(cudaMemcpyAsync(f64, d64, n_f64 * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (n_u16) CK(cudaMemcpyAsync(u16, d16, n_u16 * sizeof(uint16_t), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return 0;
  }();
  cudaStreamSynchronize(s);
  for (void* q : allocs) cudaFree(q);
  cudaStreamDestroy(s);
  return rc;
}

static_assert(B2G_GG_PLANES == GG_PLANES && B2G_GG_A_ALIGN4 == GG_A_ALIGN4 && B2G_GG_MN_MAJOR == GG_MN_MAJOR &&
                  B2G_GG_A_ROWLANES == GG_A_ROWLANES,
              "the public gg_tc flag values follow common.cuh");

namespace {
// One offset table of a gg_tc problem: its host values, how many of them the problem uses (len) and how many the kernel reads
// (reach >= len: the K-major plane producers fetch the r tables a whole 64-row chunk at a time).
struct TcTab {
  const char* name = "";
  int64_t off = -1;
  int len = 0, reach = 0;
  const int32_t* v = nullptr;
};

// The memory contracts of gg_tc_kernel that hold only by construction at each SAC call site, checked for one caller-described
// problem (the refusals are listed with b2g_debug_gg_tc in b200grasp.h).  0, or B2G_EINVAL with the broken contract named.
int check_gg_tc_problem(int idx, const b2g_debug_gg_tc_problem& p, int64_t n_f32, int64_t n_u16, const int32_t* tabs, int64_t n_tabs) {
  const std::string at = "problem " + std::to_string(idx) + ": ";
  auto fail = [&](const std::string& why) { return b2g_fail(B2G_EINVAL, at + why); };
  const int f = p.flags;
  const int allowed = GG_A_RVEC | GG_B_RVEC | GG_EPI_BIAS_RELU | GG_EPI_MASK | GG_EPI_ATOMIC | GG_COLSUM | GG_PLANES | GG_A_ALIGN4 |
                      GG_MN_MAJOR | GG_A_ROWLANES;
  if (f & ~allowed)
    return fail("flags " + std::to_string(f & ~allowed) + " are not implemented by gg_tc (GG_CN_AFFINE4 is derived, not given)");
  const bool planes = f & GG_PLANES, mn = f & GG_MN_MAJOR, al4 = f & GG_A_ALIGN4;
  if (!planes && (f & (GG_A_ALIGN4 | GG_MN_MAJOR | GG_A_ROWLANES)))
    return fail("GG_A_ALIGN4, GG_MN_MAJOR and GG_A_ROWLANES select plane producers; they need GG_PLANES");
  if ((f & GG_COLSUM) && (f & (GG_B_RVEC | GG_PLANES)))
    return fail("GG_COLSUM sums the fp32 n-direction B loads; it cannot take GG_B_RVEC or GG_PLANES");
  if (p.M < 1 || p.N < 1 || p.R < 1) return fail("M, N and R must be >= 1");
  if (p.splitR < 1 || p.splitR > p.R) return fail("splitR must be in 1..R");
  if (p.splitR > 1 && !(f & GG_EPI_ATOMIC)) return fail("splitR > 1 needs GG_EPI_ATOMIC (the splits would overwrite each other)");
  if ((p.C_hi >= 0) != (p.C_lo >= 0)) return fail("C_hi and C_lo go together");
  if ((f & GG_EPI_ATOMIC) && p.C_hi >= 0) return fail("C_hi / C_lo would hold one split's partial under GG_EPI_ATOMIC");
  const bool need_bias = f & GG_EPI_BIAS_RELU, need_mask = f & GG_EPI_MASK;
  if (p.C < 0) return fail("C is required");
  if (need_bias != (p.bias >= 0)) return fail(need_bias ? "the bias epilogue needs bias" : "bias given without a bias epilogue");
  if (need_mask != (p.mask >= 0)) return fail(need_mask ? "the mask epilogue needs mask" : "mask given without a mask epilogue");
  if (((f & GG_COLSUM) != 0) != (p.colsum >= 0)) return fail("colsum goes with GG_COLSUM");
  const bool have_planes = p.A_hi >= 0 && p.A_lo >= 0 && p.B_hi >= 0 && p.B_lo >= 0;
  const bool any_plane = p.A_hi >= 0 || p.A_lo >= 0 || p.B_hi >= 0 || p.B_lo >= 0;
  if (planes && (!have_planes || p.A >= 0 || p.B >= 0)) return fail("GG_PLANES reads A_hi, A_lo, B_hi and B_lo, not A and B");
  if (!planes && (p.A < 0 || p.B < 0 || any_plane)) return fail("fp32 problems read A and B, not planes");
  if ((p.bR_p >= 0 || p.bN_p >= 0) && (!planes || mn)) return fail("bR_p / bN_p are read by K-major plane problems only");
  // vector stores of the epilogue (float4 C and mask, uint2 C_hi / C_lo) start at the region's offset plus multiples of 4
  if (p.C % 4 || (need_mask && p.mask % 4) || (p.C_hi >= 0 && (p.C_hi % 4 || p.C_lo % 4)))
    return fail("C, mask, C_hi and C_lo must start 16-byte (C_hi / C_lo: 8-byte) aligned (the vector epilogue stores)");
  // tables: K-major plane problems read their r tables (aR, and bR_p or bR) up to index 64 ceil(R / 64) - 8
  const int rk = planes && !mn ? (p.R + GG_TC_BK - 1) / GG_TC_BK * GG_TC_BK - 7 : p.R;
  TcTab t[10];
  const int64_t offs[10] = {p.aM, p.aR, p.bR, p.bN, p.cM, p.cN, p.kM, p.kN, p.bR_p, p.bN_p};
  const char* names[10] = {"aM", "aR", "bR", "bN", "cM", "cN", "kM", "kN", "bR_p", "bN_p"};
  const int lens[10] = {p.M, p.R, p.R, p.N, p.M, p.N, p.M, p.N, p.R, p.N};
  for (int i = 0; i < 10; ++i) {
    t[i].name = names[i]; t[i].off = offs[i]; t[i].len = t[i].reach = lens[i];
    if (offs[i] < 0) {
      if (i < 6) return fail(std::string(names[i]) + " is required");
      continue;
    }
    t[i].v = tabs + offs[i];
  }
  for (int i : {6, 7}) if (!t[i].v) t[i] = t[i - 2];            // kM / kN default to cM / cN
  const TcTab &aM = t[0], &aR = t[1], &bR = t[2], &bN = t[3], &cM = t[4], &cN = t[5], &kM = t[6], &kN = t[7];
  TcTab bRk = t[8].v ? t[8] : bR, bNk = t[9].v ? t[9] : bN;    // the K-major plane B's own tables
  TcTab aRk = aR;
  if (planes && !mn) { aRk.reach = rk; bRk.reach = rk; }
  for (const TcTab* q : std::initializer_list<const TcTab*>{&aM, &aR, &bR, &bN, &cM, &cN, &kM, &kN, &aRk, &bRk, &bNk})
    if (q->off + q->reach > n_tabs) return fail(std::string(q->name) + " runs past the end of tabs");
  // [lo, hi] of the elements a table addresses; MN-major plane problems copy 8 elements from every 8-group start of aM / bN
  auto span = [](const TcTab& q, int g8) {
    int64_t lo = INT64_MAX, hi = INT64_MIN;
    for (int i = 0; i < q.len; i += g8 ? 8 : 1) { lo = std::min<int64_t>(lo, q.v[i]); hi = std::max<int64_t>(hi, q.v[i] + (g8 ? 7 : 0)); }
    return std::make_pair(lo, hi);
  };
  auto in = [&](const char* what, int64_t base, std::pair<int64_t, int64_t> x, std::pair<int64_t, int64_t> y, int64_t n) {
    return base + x.first + y.first >= 0 && base + x.second + y.second < n ? 0 : fail(std::string(what) + " reaches outside its arena");
  };
  const auto zero = std::make_pair<int64_t, int64_t>(0, 0);
  if (!planes) {
    if (int rc = in("A[aM + aR]", p.A, span(aM, 0), span(aR, 0), n_f32)) return rc;
    if (int rc = in("B[bR + bN]", p.B, span(bR, 0), span(bN, 0), n_f32)) return rc;
  } else {
    const auto sa = span(aM, mn), sb = mn ? span(bN, 1) : span(bNk, 0), ra = span(aR, 0), rb = mn ? span(bR, 0) : span(bRk, 0);
    for (int64_t base : {p.A_hi, p.A_lo}) if (int rc = in("A_hi / A_lo[aM + aR]", base, sa, ra, n_u16)) return rc;
    for (int64_t base : {p.B_hi, p.B_lo}) if (int rc = in("B_hi / B_lo[bR + bN]", base, rb, sb, n_u16)) return rc;
  }
  if (int rc = in("C[cM + cN]", p.C, span(cM, 0), span(cN, 0), n_f32)) return rc;
  if (p.C_hi >= 0)
    for (int64_t base : {p.C_hi, p.C_lo}) if (int rc = in("C_hi / C_lo[cM + cN]", base, span(cM, 0), span(cN, 0), n_u16)) return rc;
  if (need_bias) if (int rc = in("bias[n]", p.bias, zero, std::make_pair<int64_t, int64_t>(0, p.N - 1), n_f32)) return rc;
  if (need_mask) if (int rc = in("mask[kM + kN]", p.mask, span(kM, 0), span(kN, 0), n_f32)) return rc;
  if (f & GG_COLSUM) if (int rc = in("colsum[n]", p.colsum, zero, std::make_pair<int64_t, int64_t>(0, p.N - 1), n_f32)) return rc;
  // w-groups of table g (entries [w k, w k + w)) read with one vector load: contiguous, and base + the group's first offset + every
  // offset of the other side a multiple of `align` elements of `eb` bytes.  partial: a last group shorter than w is loaded too
  // (its valid part).
  auto groups = [&](const char* what, int64_t base, const TcTab& g, const TcTab& other, int w, int align, int eb, bool partial) {
    bool any = false;
    for (int i = 0; i < g.len; i += w) {
      if (!partial && i + w > g.len) break;
      any = true;
      for (int j = 1; j < w && i + j < g.len; ++j)
        if (g.v[i + j] != g.v[i] + j)
          return fail(std::string(what) + ": " + g.name + " is not contiguous in the " + std::to_string(w) + "-group at " + std::to_string(i));
      if ((base + g.v[i] + other.v[0]) % align)
        return fail(std::string(what) + ": the " + std::to_string(w) + "-groups of " + g.name + " are not " + std::to_string(align * eb) +
                    "-byte aligned");
    }
    if (any)
      for (int j = 0; j < other.len; ++j)
        if ((base + g.v[0] + other.v[j]) % align)
          return fail(std::string(what) + ": the " + std::to_string(w) + "-groups of " + g.name + " are not aligned at every " + other.name);
    return 0;
  };
  if (!planes) {        // float4 loads of full 4-groups (16 bytes of fp32)
    if (int rc = (f & GG_A_RVEC) ? groups("GG_A_RVEC", p.A, aR, aM, 4, 4, 4, false) : groups("m-direction A", p.A, aM, aR, 4, 4, 4, false))
      return rc;
    if (int rc = (f & GG_B_RVEC) ? groups("GG_B_RVEC", p.B, bR, bN, 4, 4, 4, false) : groups("n-direction B", p.B, bN, bR, 4, 4, 4, false))
      return rc;
    // int4 loads of the r tables of m- / n-direction operands (and of bR beside an m-direction A)
    if (!(f & GG_A_RVEC) && p.aR % 4) return fail("aR must start 16-byte aligned (int4 table loads)");
    if (!((f & GG_A_RVEC) && (f & GG_B_RVEC)) && p.bR % 4) return fail("bR must start 16-byte aligned (int4 table loads)");
  } else {              // cp.async of 8-groups of BF16 (16 bytes; two 8-byte halves of A under GG_A_ALIGN4)
    const int aal = al4 ? 4 : 8;
    for (int64_t base : {p.A_hi, p.A_lo})
      if (int rc = mn ? groups("MN-major A", base, aM, aR, 8, aal, 2, true) : groups("K-major A", base, aR, aM, 8, aal, 2, true)) return rc;
    for (int64_t base : {p.B_hi, p.B_lo})
      if (int rc = mn ? groups("MN-major B", base, bN, bR, 8, 8, 2, true) : groups("K-major B", base, bRk, bNk, 8, 8, 2, true)) return rc;
  }
  return 0;
}
}  // namespace

extern "C" int b2g_debug_gg_tc(int x3, const b2g_debug_gg_tc_problem* p, int n, float* f32, int64_t n_f32, uint16_t* u16, int64_t n_u16,
                               const int32_t* tabs, int64_t n_tabs) {
  if (x3 != 0 && x3 != 1) return b2g_fail(B2G_EINVAL, "x3 must be 0 (hi*hi) or 1 (hi*hi + hi*lo + lo*hi)");
  if (!p || n < 1 || n > GG_TC_MAX_DESCS) return b2g_fail(B2G_EINVAL, "1 to 16 problems per launch");
  const int64_t lim = (int64_t)1 << 31;
  if (n_f32 < 0 || n_u16 < 0 || n_tabs < 0 || n_f32 >= lim || n_u16 >= lim || n_tabs >= lim)
    return b2g_fail(B2G_EINVAL, "arena lengths must be in 0 .. 2^31 - 1");
  if ((n_f32 && !f32) || (n_u16 && !u16) || (n_tabs && !tabs)) return b2g_fail(B2G_EINVAL, "NULL arena");
  auto kernel_of = [](int f) { return (f & GG_PLANES) ? GG_PLANES : f & (GG_A_RVEC | GG_B_RVEC); };
  for (int i = 1; i < n; ++i)
    if (kernel_of(p[i].flags) != kernel_of(p[0].flags))
      return b2g_fail(B2G_EINVAL, "problem " + std::to_string(i) +
                                      ": its flags select another gg_tc kernel than problem 0's (GG_PLANES, else GG_A_RVEC | GG_B_RVEC)");
  for (int i = 0; i < n; ++i)
    if (int rc = check_gg_tc_problem(i, p[i], n_f32, n_u16, tabs, n_tabs)) return rc;

  int num_sms = 0;
  if (int rc = check_device(0, &num_sms)) return rc;
  cudaStream_t s = nullptr;
  CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  std::vector<void*> allocs;
  const int rc = [&]() -> int {
    float* d32 = nullptr; uint16_t* d16 = nullptr; int32_t* dt = nullptr;
    if (int rc = dev_alloc(allocs, s, &d32, n_f32, false)) return rc;
    if (int rc = dev_alloc(allocs, s, &d16, n_u16, false)) return rc;
    if (int rc = dev_alloc(allocs, s, &dt, n_tabs, false)) return rc;
    if (n_f32) CK(cudaMemcpyAsync(d32, f32, n_f32 * sizeof(float), cudaMemcpyHostToDevice, s));
    if (n_u16) CK(cudaMemcpyAsync(d16, u16, n_u16 * sizeof(uint16_t), cudaMemcpyHostToDevice, s));
    if (n_tabs) CK(cudaMemcpyAsync(dt, tabs, n_tabs * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    // host copies of the epilogue tables under their device addresses, as the SAC handle keeps them, for gg_tc_columns
    std::map<const int*, std::vector<int>> host_tabs;
    auto keep = [&](int64_t off, int len) {
      if (off < 0) return;
      std::vector<int>& v = host_tabs[dt + off];
      if ((int)v.size() < len) v.assign(tabs + off, tabs + off + len);
    };
    ColIds col_ids;
    GemmGroup g;
    g.name = "debug_gg_tc";
    g.tc = true;
    auto f32p = [&](int64_t off) { return off >= 0 ? d32 + off : nullptr; };
    auto u16p = [&](int64_t off) { return off >= 0 ? d16 + off : nullptr; };
    auto tabp = [&](int64_t off) -> const int* { return off >= 0 ? dt + off : nullptr; };
    for (int i = 0; i < n; ++i) {
      const b2g_debug_gg_tc_problem& q = p[i];
      keep(q.cM, q.M); keep(q.cN, q.N); keep(q.kM, q.M); keep(q.kN, q.N);
      GemmDesc d = gemm_desc(f32p(q.A), tabp(q.aM), tabp(q.aR), f32p(q.B), tabp(q.bR), tabp(q.bN), d32 + q.C, tabp(q.cM), tabp(q.cN),
                             q.M, q.N, q.R, q.flags, q.splitR);
      d.kM = tabp(q.kM); d.kN = tabp(q.kN);
      d.bias = f32p(q.bias); d.mask = f32p(q.mask); d.colsum = f32p(q.colsum);
      d.A_hi = u16p(q.A_hi); d.A_lo = u16p(q.A_lo); d.B_hi = u16p(q.B_hi); d.B_lo = u16p(q.B_lo);
      d.bR_p = tabp(q.bR_p); d.bN_p = tabp(q.bN_p);
      d.C_hi = u16p(q.C_hi); d.C_lo = u16p(q.C_lo);
      g.host.push_back(d);
    }
    for (auto& d : g.host) gg_tc_columns(d, host_tabs, col_ids);
    if (int rc = finalize_tiles(g, allocs, s, GG_TC_BM, GG_TC_BN)) return rc;
    CK(gg_tc_launch(g.host.data(), n, g.total_tiles, g.host[0].flags, x3, num_sms, s));
    if (n_f32) CK(cudaMemcpyAsync(f32, d32, n_f32 * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (n_u16) CK(cudaMemcpyAsync(u16, d16, n_u16 * sizeof(uint16_t), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return 0;
  }();
  cudaStreamSynchronize(s);
  for (void* q : allocs) cudaFree(q);
  cudaStreamDestroy(s);
  return rc;
}
