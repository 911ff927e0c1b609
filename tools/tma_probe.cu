// tma_probe: checks, on a real H100, every cp.async.bulk.tensor (TMA) behaviour the conv engine relies on BEFORE the
// engine is built on it.  Each case encodes a tensor map over a device buffer holding element-index values, issues
// one tiled load into shared memory, copies the tile back and compares it with the layout the kernel expects:
//   1. 2-D tile, SWIZZLE_128B: row r, 16-byte chunk c lands at r*128 + ((c ^ (r & 7)) << 4)      (wgmma K-major tile)
//   2. 4-D view with OVERLAPPING strides + element strides {1,2,2,1}: implicit im2col of a stride-2 4x4 conv
//   3. negative start coordinates / out-of-bound rows are zero-filled and still complete the full-box byte count
//   4. 5-D view of a 1-channel image (8x8 patch, stride 4, pair-of-output-pixel dimension with a 16-byte stride)
//   5. tensor map resident in GLOBAL memory (table of maps) instead of a __grid_constant__ parameter
//   6. TMA store (shared -> global) of a swizzled tile
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O2 -o tools/tma_probe tools/tma_probe.cu ; run on the GPU.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(2); } } while (0)

typedef CUresult (*EncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiled g_encode = nullptr;

static bool make_map(CUtensorMap* m, void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                     const uint32_t* estr, CUtensorMapSwizzle sw) {
  cuuint64_t gd[5], gs[5];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = estr[i]; }
  for (int i = 0; i + 1 < rank; ++i) gs[i] = strides_bytes[i];
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, base, gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { printf("  cuTensorMapEncodeTiled failed: %d\n", (int)r); return false; }
  return true;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// loads one box at coords c[0..rank) into smem (1024-aligned), copies `bytes` back to out; flag = 1 if the mbarrier completed
__global__ void load_kernel(const __grid_constant__ CUtensorMap pmap, const CUtensorMap* gmap, int use_global, int rank, int c0, int c1, int c2,
                            int c3, int c4, int bytes, uint8_t* out, int* flag) {
  extern __shared__ uint8_t raw[];
  __shared__ __align__(8) uint64_t bar;
  const uint32_t tile = (smem_u32(raw) + 1023u) & ~1023u;
  uint8_t* tile_p = raw + (tile - smem_u32(raw));
  for (int i = threadIdx.x; i < bytes; i += blockDim.x) tile_p[i] = 0xCD;
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    const void* mp = use_global ? (const void*)gmap : (const void*)&pmap;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar)), "r"(bytes) : "memory");
    const uint32_t b = smem_u32(&bar);
    if (rank == 2)
      asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(tile),
                   "l"(mp), "r"(b), "r"(c0), "r"(c1)
                   : "memory");
    else if (rank == 4)
      asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(tile),
                   "l"(mp), "r"(b), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
                   : "memory");
    else
      asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(
                       tile),
                   "l"(mp), "r"(b), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
                   : "memory");
    int ok = 0;
    for (int spin = 0; spin < (1 << 20) && !ok; ++spin) {
      asm volatile(
          "{\n\t.reg .pred p;\n\t"
          "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
          "selp.b32 %0, 1, 0, p;\n\t}"
          : "=r"(ok)
          : "r"(b)
          : "memory");
    }
    *flag = ok;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < bytes; i += blockDim.x) out[i] = tile_p[i];
}

// smem tile (filled with element values by the threads, swizzled like a TMA load would) -> global through a 2-D map
__global__ void store_kernel(const __grid_constant__ CUtensorMap pmap, int rows, int c0, int c1) {
  extern __shared__ uint8_t raw[];
  const uint32_t tile = (smem_u32(raw) + 1023u) & ~1023u;
  uint16_t* tp = (uint16_t*)(raw + (tile - smem_u32(raw)));
  for (int i = threadIdx.x; i < rows * 64; i += blockDim.x) {
    const int r = i / 64, e = i % 64, ch = e / 8;
    tp[(r * 128 + ((ch ^ (r & 7)) << 4)) / 2 + (e % 8)] = (uint16_t)(0x4000 + i);
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(&pmap), "r"(tile), "r"(c0), "r"(c1) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
}

static int run_load(const CUtensorMap& m, const CUtensorMap* dmap, int use_global, int rank, const int* c, int bytes, std::vector<uint16_t>& host) {
  uint8_t* dout;
  int* dflag;
  CK(cudaMalloc(&dout, bytes));
  CK(cudaMalloc(&dflag, 4));
  CK(cudaMemset(dflag, 0, 4));
  CK(cudaFuncSetAttribute(load_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
  load_kernel<<<1, 128, bytes + 2048>>>(m, dmap, use_global, rank, c[0], c[1], c[2], c[3], c[4], bytes, dout, dflag);
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("  kernel failed: %s\n", cudaGetErrorString(e)); exit(3); }
  int flag = 0;
  CK(cudaMemcpy(&flag, dflag, 4, cudaMemcpyDeviceToHost));
  host.resize(bytes / 2);
  CK(cudaMemcpy(host.data(), dout, bytes, cudaMemcpyDeviceToHost));
  cudaFree(dout); cudaFree(dflag);
  return flag;
}

// value stored at element index i of a probe buffer: a bf16 bit pattern that is unique for i < 2^15 and never 0 / 0xCDCD
static inline uint16_t val(size_t i) { return (uint16_t)(0x4000 + (i & 0x3FFF)); }

int main(int argc, char** argv) {
  const int only = argc > 1 ? atoi(argv[1]) : 0;   // 0 = the cases the engine relies on (1-3, 5, 6); 4, 7, 8, 9 = exploratory, one per process
  CK(cudaSetDevice(0));
  CK(cudaFree(0));
  cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void**)&g_encode, cudaEnableDefault, &q));
  if (!g_encode || q != cudaDriverEntryPointSuccess) { printf("no cuTensorMapEncodeTiled\n"); return 2; }
  int fails = 0;
  const size_t NEL = 1 << 20;
  std::vector<uint16_t> src(NEL);
  for (size_t i = 0; i < NEL; ++i) src[i] = val(i);
  uint16_t* d;
  CK(cudaMalloc(&d, NEL * 2));
  CK(cudaMemcpy(d, src.data(), NEL * 2, cudaMemcpyHostToDevice));
  std::vector<uint16_t> got;
  auto sw_off = [](int r, int ch) { return r * 128 + ((ch ^ (r & 7)) << 4); };   // bytes

  if (only == 0 || only == 1) {   // ---- case 1: 2-D [rows=256][cols=512] bf16, box {64, 128}, SW128
    printf("case 1: 2-D tile, SWIZZLE_128B\n");
    CUtensorMap m;
    const uint64_t dims[2] = {512, 256}, str[1] = {512 * 2};
    const uint32_t box[2] = {64, 128}, es[2] = {1, 1};
    if (!make_map(&m, d, 2, dims, str, box, es, CU_TENSOR_MAP_SWIZZLE_128B)) { ++fails; }
    else {
      const int c[5] = {128, 64, 0, 0, 0};
      const int flag = run_load(m, nullptr, 0, 2, c, 128 * 128, got);
      int bad = 0;
      for (int r = 0; r < 128; ++r)
        for (int e = 0; e < 64; ++e) {
          const uint16_t exp = val((size_t)(64 + r) * 512 + 128 + e);
          if (got[(sw_off(r, e / 8)) / 2 + (e % 8)] != exp) ++bad;
        }
      printf("  completed=%d mismatches=%d\n", flag, bad);
      if (!flag || bad) ++fails;
    }
  }
  if (only == 0 || only == 2) {   // ---- case 2: h1 [B=8][15][15][32] bf16 viewed as {64 (two pixels x 32 ch), 14 (x), 15 (y), B}; strides {64 B, 15*64 B, 225*64 B}
    printf("case 2: 4-D overlapping-stride view, element strides {1,2,2,1} (conv2 implicit im2col)\n");
    CUtensorMap m;
    const uint64_t dims[4] = {64, 14, 15, 8}, str[3] = {64, 15 * 64, 225 * 64};
    const uint32_t box[4] = {64, 12, 12, 3}, es[4] = {1, 2, 2, 1};
    if (!make_map(&m, d, 4, dims, str, box, es, CU_TENSOR_MAP_SWIZZLE_128B)) { ++fails; }
    else {
      for (int kpos = 0; kpos < 3; ++kpos) {
        const int kx0 = (kpos & 1) * 2, ky = kpos + 1, b0 = 2;
        const int c[5] = {0, kx0, ky, b0, 0};
        const int rows = 3 * 36;
        const int flag = run_load(m, nullptr, 0, 4, c, rows * 128, got);
        int bad = 0;
        for (int bb = 0; bb < 3; ++bb)
          for (int oy = 0; oy < 6; ++oy)
            for (int ox = 0; ox < 6; ++ox)
              for (int e = 0; e < 64; ++e) {
                const int r = (bb * 6 + oy) * 6 + ox;
                const size_t gi = ((size_t)((b0 + bb) * 15 + (2 * oy + ky)) * 15 + (2 * ox + kx0)) * 32 + e;
                if (got[(sw_off(r, e / 8)) / 2 + (e % 8)] != val(gi)) ++bad;
              }
        printf("  (ky=%d,kx0=%d): completed=%d mismatches=%d of %d\n", ky, kx0, flag, bad, rows * 64);
        if (!flag || bad) ++fails;
      }
    }
  }
  if (only == 0 || only == 3) {   // ---- case 3: dZ3 [B=8][4][4][64]; box {64, 6, 6, 3} starting at (0, -kx, -ky, b0): zero fill outside, batch overrun at the end
    printf("case 3: negative coordinates / OOB zero fill (conv3 dgrad view)\n");
    CUtensorMap m;
    const uint64_t dims[4] = {64, 4, 4, 8}, str[3] = {128, 4 * 128, 16 * 128};
    const uint32_t box[4] = {64, 6, 6, 3}, es[4] = {1, 1, 1, 1};
    if (!make_map(&m, d, 4, dims, str, box, es, CU_TENSOR_MAP_SWIZZLE_128B)) { ++fails; }
    else {
      for (int t = 0; t < 2; ++t) {
        const int kx = t ? 2 : 1, ky = t ? 0 : 2, b0 = t ? 6 : 1;      // t = 1: samples 6,7,8 -> the last one is out of range
        const int c[5] = {0, -kx, -ky, b0, 0};
        const int rows = 3 * 36;
        const int flag = run_load(m, nullptr, 0, 4, c, rows * 128, got);
        int bad = 0;
        for (int bb = 0; bb < 3; ++bb)
          for (int y = 0; y < 6; ++y)
            for (int x = 0; x < 6; ++x)
              for (int e = 0; e < 64; ++e) {
                const int r = (bb * 6 + y) * 6 + x, sy = y - ky, sx = x - kx, b = b0 + bb;
                uint16_t exp = 0;
                if (sy >= 0 && sy < 4 && sx >= 0 && sx < 4 && b < 8) exp = val(((size_t)(b * 4 + sy) * 4 + sx) * 64 + e);
                if (got[(sw_off(r, e / 8)) / 2 + (e % 8)] != exp) ++bad;
              }
        printf("  (ky=%d,kx=%d,b0=%d): completed=%d mismatches=%d\n", ky, kx, b0, flag, bad);
        if (!flag || bad) ++fails;
      }
    }
  }
  if (only == 4) {   // ---- case 4: image [B=4][64][64] (1 channel), patch view {8 kx, 8 ky, 8 j (pairs of output pixels: 16 B), 15 oy (4 rows), B}
    printf("case 4: 5-D view of a 1-channel image (conv1: 8x8 patches, stride 4, even output columns)\n");
    CUtensorMap m;
    const uint64_t dims[5] = {8, 8, 8, 15, 4}, str[4] = {64 * 2, 8 * 2, 4 * 64 * 2, 4096 * 2};
    const uint32_t box[5] = {8, 8, 8, 15, 1}, es[5] = {1, 1, 1, 1, 1};
    for (int par = 0; par < 2; ++par) {
      // odd output columns: the same view over a copy of the image shifted by 4 pixels (8 bytes) -- here emulated by a
      // base pointer 4 elements further, which is only legal when that address is 16-byte aligned: expected to FAIL
      // for par = 1 on the unshifted buffer (documented), so the engine keeps a second, shifted copy of the planes.
      void* base = (void*)(d + (par ? 4 : 0));
      printf("  parity %d (base %s16-byte aligned): ", par, ((uintptr_t)base & 15) ? "NOT " : "");
      if (!make_map(&m, base, 5, dims, str, box, es, CU_TENSOR_MAP_SWIZZLE_128B)) { if (!par) ++fails; continue; }
      const int c[5] = {0, 0, 0, 0, 2};
      const int rows = 120;
      const int flag = run_load(m, nullptr, 0, 5, c, rows * 128, got);
      int bad = 0;
      for (int oy = 0; oy < 15; ++oy)
        for (int j = 0; j < 8; ++j)
          for (int ky = 0; ky < 8; ++ky)
            for (int kx = 0; kx < 8; ++kx) {
              const int r = oy * 8 + j, e = ky * 8 + kx;
              const size_t gi = (size_t)2 * 4096 + (size_t)(4 * oy + ky) * 64 + 8 * j + kx + (par ? 4 : 0);
              if (got[(sw_off(r, e / 8)) / 2 + (e % 8)] != val(gi)) ++bad;
            }
      printf("completed=%d mismatches=%d\n", flag, bad);
      if (!flag || bad) ++fails;
    }
  }
  if (only == 0 || only == 5) {   // ---- case 5: map in global memory
    printf("case 5: tensor map resident in global memory\n");
    CUtensorMap m, *dm;
    const uint64_t dims[2] = {512, 256}, str[1] = {512 * 2};
    const uint32_t box[2] = {64, 64}, es[2] = {1, 1};
    if (!make_map(&m, d, 2, dims, str, box, es, CU_TENSOR_MAP_SWIZZLE_128B)) { ++fails; }
    else {
      CK(cudaMalloc(&dm, 4 * sizeof(CUtensorMap)));
      CK(cudaMemcpy(dm + 2, &m, sizeof(m), cudaMemcpyHostToDevice));
      const int c[5] = {64, 32, 0, 0, 0};
      const int flag = run_load(m, dm + 2, 1, 2, c, 64 * 128, got);
      int bad = 0;
      for (int r = 0; r < 64; ++r)
        for (int e = 0; e < 64; ++e)
          if (got[(sw_off(r, e / 8)) / 2 + (e % 8)] != val((size_t)(32 + r) * 512 + 64 + e)) ++bad;
      printf("  completed=%d mismatches=%d\n", flag, bad);
      if (!flag || bad) ++fails;
    }
  }
  if (only == 0 || only == 6) {   // ---- case 6: TMA store of a swizzled 32-row tile into a [256][512] tensor, partly out of range (rows clipped)
    printf("case 6: TMA store (shared -> global), rows beyond the tensor are clipped\n");
    uint16_t* o;
    CK(cudaMalloc(&o, 256 * 512 * 2));
    CK(cudaMemset(o, 0, 256 * 512 * 2));
    CUtensorMap m;
    const uint64_t dims[2] = {512, 240}, str[1] = {512 * 2};      // only 240 rows are "inside"
    const uint32_t box[2] = {64, 32}, es[2] = {1, 1};
    if (!make_map(&m, o, 2, dims, str, box, es, CU_TENSOR_MAP_SWIZZLE_128B)) { ++fails; }
    else {
      CK(cudaFuncSetAttribute(store_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
      store_kernel<<<1, 128, 8192>>>(m, 32, 192, 224);
      cudaError_t e = cudaDeviceSynchronize();
      if (e != cudaSuccess) { printf("  store kernel failed: %s\n", cudaGetErrorString(e)); return 3; }
      std::vector<uint16_t> h(256 * 512);
      CK(cudaMemcpy(h.data(), o, h.size() * 2, cudaMemcpyDeviceToHost));
      int bad = 0, outside = 0;
      for (int r = 0; r < 256; ++r)
        for (int cc = 0; cc < 512; ++cc) {
          const bool in = r >= 224 && r < 240 && cc >= 192 && cc < 256;
          const uint16_t exp = in ? (uint16_t)(0x4000 + (r - 224) * 64 + (cc - 192)) : 0;
          if (h[(size_t)r * 512 + cc] != exp) { ++bad; if (!in) ++outside; }
        }
      printf("  mismatches=%d (outside the box / clipped rows: %d)\n", bad, outside);
      if (bad) ++fails;
    }
  }
  if (only == 7) {   // ---- case 7: 3-D view with NON-MONOTONIC strides {kx 2 B, ky 128 B, j 16 B} (rank 3)
    printf("case 7: 3-D non-monotonic strides\n");
    CUtensorMap m;
    const uint64_t dims[3] = {8, 8, 8}, str[2] = {128, 16};
    const uint32_t box[3] = {8, 8, 8}, es[3] = {1, 1, 1};
    if (!make_map(&m, d, 3, dims, str, box, es, CU_TENSOR_MAP_SWIZZLE_128B)) ++fails;
    else {
      CUtensorMap* dm; CK(cudaMalloc(&dm, sizeof(m))); CK(cudaMemcpy(dm, &m, sizeof(m), cudaMemcpyHostToDevice));
      const int c[5] = {0, 0, 0, 0, 0};
      // rank-3 loads go through the 4-D path of the probe kernel with a unit 4th coordinate: not available -> use rank 2 fallback? no: issue as 5-D is wrong.
      printf("  (encode ok)\n");
    }
  }
  if (only == 8) {   // ---- case 8: 5-D view, plain contiguous (monotonic) strides
    printf("case 8: 5-D contiguous tensor\n");
    CUtensorMap m;
    const uint64_t dims[5] = {64, 4, 4, 4, 4}, str[4] = {128, 512, 2048, 8192};
    const uint32_t box[5] = {64, 2, 2, 2, 2}, es[5] = {1, 1, 1, 1, 1};
    if (!make_map(&m, d, 5, dims, str, box, es, CU_TENSOR_MAP_SWIZZLE_128B)) ++fails;
    else {
      const int c[5] = {0, 1, 1, 1, 1};
      const int flag = run_load(m, nullptr, 0, 5, c, 16 * 128, got);
      int bad = 0, r = 0;
      for (int i4 = 0; i4 < 2; ++i4) for (int i3 = 0; i3 < 2; ++i3) for (int i2 = 0; i2 < 2; ++i2) for (int i1 = 0; i1 < 2; ++i1, ++r)
        for (int e = 0; e < 64; ++e) {
          const size_t gi = (size_t)(1 + i4) * 4096 + (1 + i3) * 1024 + (1 + i2) * 256 + (1 + i1) * 64 + e;
          if (got[(sw_off(r, e / 8)) / 2 + (e % 8)] != val(gi)) ++bad;
        }
      printf("  completed=%d mismatches=%d\n", flag, bad);
      if (!flag || bad) ++fails;
    }
  }
  if (only == 9) {   // ---- case 9: conv1 through a space-to-depth image [b][16][16][16] : {32 = 2 px x 16, 2 dy (512 B), 15 ox (32 B), 15 oy (512 B), b}
    printf("case 9: 5-D space-to-depth conv1 view (non-monotonic, repeated strides)\n");
    CUtensorMap m;
    const uint64_t dims[5] = {32, 2, 15, 15, 4}, str[4] = {512, 32, 512, 8192};
    const uint32_t box[5] = {32, 2, 15, 8, 1}, es[5] = {1, 1, 1, 1, 1};
    if (!make_map(&m, d, 5, dims, str, box, es, CU_TENSOR_MAP_SWIZZLE_128B)) ++fails;
    else {
      const int c[5] = {0, 0, 0, 0, 1};
      const int rows = 120;
      const int flag = run_load(m, nullptr, 0, 5, c, rows * 128, got);
      int bad = 0;
      for (int oy = 0; oy < 8; ++oy) for (int ox = 0; ox < 15; ++ox) for (int dy = 0; dy < 2; ++dy) for (int e = 0; e < 32; ++e) {
        const int r = oy * 15 + ox, ee = dy * 32 + e;
        const size_t gi = (size_t)4096 + (size_t)(oy + dy) * 256 + ox * 16 + e;
        if (got[(sw_off(r, ee / 8)) / 2 + (ee % 8)] != val(gi)) ++bad;
      }
      printf("  completed=%d mismatches=%d\n", flag, bad);
      if (!flag || bad) ++fails;
    }
  }
  printf("tma_probe: %s (%d failing cases)\n", fails ? "FAIL" : "ALL OK", fails);
  return fails ? 1 : 0;
}
