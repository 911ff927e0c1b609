// tma_rate: how fast can ONE SM (and all 132 of an H100 together) pull L2-resident data with cp.async.bulk.tensor?
// Each CTA streams `iters` boxes of [rows x 128 B] from a 32 MB bf16 matrix (L2 resident after the warm-up pass) into a ring of
// `stages` shared-memory slots; a box is re-armed as soon as it lands (no consumer).  Reports GB/s per SM and aggregate
// for several (grid, stages, rows-per-box, issuing-thread count).
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s line %d\n", cudaGetErrorString(e_), __LINE__); exit(2); } } while (0)
typedef CUresult (*EncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__global__ void __launch_bounds__(128, 1) k(const __grid_constant__ CUtensorMap map, int iters, int stages, int rows, int nrows_total, int issuers) {
  extern __shared__ uint8_t raw[];
  __shared__ __align__(8) uint64_t bar[32];
  const uint32_t ring = (smem_u32(raw) + 1023u) & ~1023u;
  const int box_bytes = rows * 128;
  if (threadIdx.x == 0) { for (int s = 0; s < stages * issuers; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar[s]))); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncthreads();
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (w < issuers && lane == 0) {
    // issuer w owns its own `stages` slots and barriers: ring slot w * stages + s
    for (int it = 0; it < iters; ++it) {
      const int s = it % stages, slot = w * stages + s;
      const int use = it / stages;
      if (use > 0) {
        const uint32_t par = (use - 1) & 1;
        asm volatile("{\n\t.reg .pred p;\n\tW:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra D;\n\tbra W;\n\tD:\n\t}" ::"r"(smem_u32(&bar[slot])), "r"(par) : "memory");
      }
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar[slot])), "r"(box_bytes) : "memory");
      const int col = ((it + w) * 64) & 1023;
      const int row = (int)(((unsigned)blockIdx.x * 977u + (unsigned)(it * 4 + w) * (unsigned)rows) % (unsigned)(nrows_total - rows));
      asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(ring + slot * box_bytes),
                   "l"(&map), "r"(smem_u32(&bar[slot])), "r"(col), "r"(row)
                   : "memory");
    }
    for (int s = 0; s < stages && s < iters; ++s) {
      const int uses = (iters - 1 - s) / stages + 1;
      const uint32_t par = (uses - 1) & 1;
      asm volatile("{\n\t.reg .pred p;\n\tW2:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra D2;\n\tbra W2;\n\tD2:\n\t}" ::"r"(smem_u32(&bar[w * stages + s])), "r"(par) : "memory");
    }
  }
}

int main() {
  CK(cudaSetDevice(0)); CK(cudaFree(0));
  EncodeTiled enc; cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void**)&enc, cudaEnableDefault, &q));
  const int NR = 16384, NC = 1024;          // 32 MB of bf16
  uint16_t* d; CK(cudaMalloc(&d, (size_t)NR * NC * 2)); CK(cudaMemset(d, 0, (size_t)NR * NC * 2));
  CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  const int rows_opts[3] = {128, 64, 32};
  for (int ri = 0; ri < 3; ++ri) {
    const int rows = rows_opts[ri];
    CUtensorMap m;
    cuuint64_t gd[2] = {NC, NR}, gs[1] = {NC * 2}; cuuint32_t bx[2] = {64, (cuuint32_t)rows}, es[2] = {1, 1};
    if (enc(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, d, gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) { printf("encode failed\n"); return 1; }
    const int grids[2] = {1, 132};
    for (int gi = 0; gi < 2; ++gi)
      for (int stages = 2; stages <= 8; stages *= 2) {
        for (int issuers = 1; issuers <= 4; issuers *= 2) {
          if (stages * issuers * rows * 128 > 200 * 1024 || stages * issuers > 32) continue;
          const int iters = 4096 / (rows / 32);
          k<<<grids[gi], 128, 200 * 1024 + 2048>>>(m, 64, stages, rows, NR, issuers);   // warm L2
          CK(cudaDeviceSynchronize());
          CK(cudaEventRecord(e0));
          k<<<grids[gi], 128, 200 * 1024 + 2048>>>(m, iters, stages, rows, NR, issuers);
          CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
          float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
          const double bytes = (double)grids[gi] * iters * issuers * rows * 128;
          printf("rows/box %3d  grid %3d  stages %2d  issuers %d : %7.1f GB/s per SM, %8.1f GB/s total\n", rows, grids[gi], stages, issuers, bytes / grids[gi] / ms / 1e6, bytes / ms / 1e6);
        }
      }
  }
  return 0;
}
