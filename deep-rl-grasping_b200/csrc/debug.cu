// Bring-up / measurement hooks of libb200grasp (not on the product path).
//
// b2g_debug_gemm: one dense C[M,N] = A[M,K] * B[N,K]^T through the wgmma gather-GEMM engine (register-staged fp32
// operands, BF16 hi/lo split when x3 != 0), used by tools/tc_accum_probe.py to measure what the tensor core's fp32
// accumulation in registers does to long, cancelling reductions -- independently of the operand split.
// b2g_debug_tensor_info / b2g_debug_tensor: one plane of one named device tensor of a SAC handle (engine v2 planes, fp32 head
// buffers) back to the host, so that tests can hold each contraction to a float64 contraction of the inputs it actually read.
#include <cuda_runtime.h>

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
