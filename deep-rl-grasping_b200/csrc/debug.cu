// Bring-up / measurement hooks of libb200grasp (not on the product path).
//
// b2g_debug_gemm: one dense C[M,N] = A[M,K] * B[N,K]^T through the wgmma gather-GEMM engine (register-staged fp32
// operands, BF16 hi/lo split when x3 != 0), used by tools/tc_accum_probe.py to measure what the tensor core's fp32
// accumulation in registers does to long, cancelling reductions -- independently of the operand split.
#include <cuda_runtime.h>

#include <string>
#include <vector>

#include "../../include/b200grasp.h"
#include "common.cuh"

using namespace b2g;

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
