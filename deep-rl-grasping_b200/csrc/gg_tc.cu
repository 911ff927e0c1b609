// wgmma gather-GEMM engine (sm_90a): the dense contractions of the SAC step on the Hopper tensor
// cores with fp32 accumulation in registers.
//
//   C[cM[m] + cN[n]] (=|+=) epi( sum_r A[aM[m] + aR[r]] * B[bR[r] + bN[n]] )       (common.cuh)
//
// Persistent, warp-specialised kernel: grid = min(#tiles, #SMs); every CTA walks the flattened tile
// list of a grouped launch (tile = 128(m) x <=64(n) x its r-range) with two concurrent roles:
//   * producer warps gather fp32 operands through the offset tables (implicit im2col / wgrad /
//     dgrad views), split every value into BF16 hi + BF16 lo (x = hi + lo to ~2^-17) and write both
//     as K-major, 128B-swizzled wgmma tiles into a 3-stage shared-memory ring that runs continuously
//     across tiles (generic-proxy stores -> fence.proxy.async -> mbarrier arrive);
//   * consumer warpgroups issue wgmma.mma_async over the ring into register accumulators: mode
//     BF16X3 = hi*hi + hi*lo + lo*hi (fp32-faithful to ~1e-5, the parity mode), mode BF16 = hi*hi
//     only (fast mode); each finished chunk frees its ring slot.  After the last chunk of a tile the
//     accumulators go to a shared-memory tile (one row per thread from there on), and the same warps
//     apply bias+ReLU / ReLU-mask / split-R atomics and store while the producers already fill the
//     ring for the next tile.
// Shared memory: 3 x 48 KiB ring, 32 KiB accumulator tile, 32 KiB store staging.
#include <cuda_bf16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace b2g {
namespace {

constexpr int TM = GG_TC_BM, TN = GG_TC_BN, TK = GG_TC_BK;   // tile: 128 x 64 x 64
constexpr int STAGES = 3;
// warp roles.  register-staged operands (fp32 sources): 16 producer warps, one consumer warpgroup (640 threads);
// BF16-plane operands (cp.async): 8 producer warps, two consumer warpgroups (512 threads).  Consumers run the MMAs and the
// epilogue; warpgroups start at a warp index that is a multiple of 4.
template <bool planes> struct Roles {
  static constexpr int NPROD = planes ? 256 : 512;
  static constexpr int MMA_WARP = NPROD / 32;            // first consumer warp
  static constexpr int NEPI = planes ? 256 : 128;
  static constexpr int NTHREADS = NPROD + NEPI;
  static constexpr int EPI_COLS = planes ? 32 : 64;      // accumulator columns handled by one consumer warp in the epilogue
  static constexpr int MB = planes ? 1 : 2;              // m64 blocks of the 128-row tile per consumer warpgroup
};
constexpr int A_BYTES = TM * TK * 2;                    // 16 KiB per (hi | lo)
constexpr int B_BYTES = TN * TK * 2;                    // 8 KiB
constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;  // 48 KiB
constexpr int STG_BYTES = TM * TN * 4;                   // fp32 output staging tile (32 KiB): coalesced epilogue stores
constexpr int ACC_BYTES = TM * TN * 4;                   // fp32 accumulator tile (32 KiB), rows of 256 B, 16-byte chunks XOR-swizzled by row
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STG_BYTES + ACC_BYTES + 1024;

struct DescPack {
  GemmDesc d[GG_TC_MAX_DESCS];
  int n;
  int total_tiles;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(bar), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// The wgmmas of one ring chunk for the MB m64 blocks of this warpgroup (rows 64 * (m_first + mb)), N = tile width rounded up to
// 32 or 64.  K-major tiles: rows of 128 B, 8-row groups 1024 B apart, 16 k = 32 bytes along the row.  MN-major tiles (wgrad):
// 8-row K atoms of two 64-element M atoms (A, 1024 B apart) or one N atom (B); 16 k = two K atoms.
template <int N, int TRANS, int MB>
__device__ __forceinline__ void mma_chunk(float (&acc)[MB][32], uint32_t sA_hi, uint32_t sA_lo, uint32_t sB_hi, uint32_t sB_lo, int m_first, int x3) {
#pragma unroll
  for (int k = 0; k < TK / 16; ++k) {
    const uint64_t bh = TRANS ? wg_desc(sB_hi + k * 2048, 1024, 1024) : wg_desc(sB_hi + k * 32, 16, 1024);
    const uint64_t bl = TRANS ? wg_desc(sB_lo + k * 2048, 1024, 1024) : wg_desc(sB_lo + k * 32, 16, 1024);
#pragma unroll
    for (int mb = 0; mb < MB; ++mb) {
      const uint32_t ao = TRANS ? (uint32_t)(k * 4096 + (m_first + mb) * 1024) : (uint32_t)((m_first + mb) * 8192 + k * 32);
      const uint64_t ah = TRANS ? wg_desc(sA_hi + ao, 1024, 2048) : wg_desc(sA_hi + ao, 16, 1024);
      Wgmma<N, TRANS>::mma(acc[mb], ah, bh);
      if (x3) {
        const uint64_t al = TRANS ? wg_desc(sA_lo + ao, 1024, 2048) : wg_desc(sA_lo + ao, 16, 1024);
        Wgmma<N, TRANS>::mma(acc[mb], ah, bl);
        Wgmma<N, TRANS>::mma(acc[mb], al, bh);
      }
    }
  }
}

// 8 fp32 -> 8 bf16 hi (4 x b32) + 8 bf16 lo.  cvt.rn.bf16x2.f32 d, a, b packs a into the upper half.
__device__ __forceinline__ void split8(const float (&x)[8], uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint32_t d;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(x[2 * i + 1]), "f"(x[2 * i]));
    const float r0 = x[2 * i] - __uint_as_float(d << 16);
    const float r1 = x[2 * i + 1] - __uint_as_float(d & 0xFFFF0000u);
    uint32_t e;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(e) : "f"(r1), "f"(r0));
    h[i] = d; l[i] = e;
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}
// byte offset of the 16-byte chunk (row, c) inside a K-major SWIZZLE_128B tile (128 B per row)
__device__ __forceinline__ uint32_t sw128(int row, int c) { return (uint32_t)(row * 128 + ((c ^ (row & 7)) << 4)); }

__device__ __forceinline__ void st_shared16(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// 16-byte (or 8-byte) asynchronous global->shared copy with zero fill beyond src_bytes
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async8(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// the mbarrier receives one arrival when all cp.async issued so far by this thread have landed
__device__ __forceinline__ void cp_async_arrive_noinc(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ float4 ldg4(const float* p) { return *reinterpret_cast<const float4*>(p); }
// Descriptor fields live in the kernel-parameter constant bank behind a run-time problem index; left alone the
// compiler re-reads them with register-indexed LDCs at every use inside the copy / store loops (hundreds of dependent
// constant loads per tile).  pin() makes a value opaque so that it stays in a register for the whole tile.
template <class T> __device__ __forceinline__ T* pin(T* p) { asm volatile("" : "+l"(p)); return p; }
__device__ __forceinline__ int pin(int v) { asm volatile("" : "+r"(v)); return v; }

struct TileInfo {
  int p, m0, n0, tm, r_begin, r_end, nchunks, un;
};
__device__ __forceinline__ TileInfo tile_info(const DescPack& pk, int tile) {
  int p = 0;
  while (p + 1 < pk.n && tile >= pk.d[p + 1].tile_start) ++p;
  const GemmDesc& d = pk.d[p];
  int t = tile - d.tile_start;
  // run-time integer divisions only where they are needed: most problems have one column block and no split-R
  const int splitR = d.splitR, tiles_n = d.tiles_n, R = d.R;
  int split = 0;
  if (splitR > 1) {
    const int per = d.tiles_m * tiles_n;
    split = t / per;
    t -= split * per;
  }
  TileInfo ti;
  ti.p = p;
  ti.tm = tiles_n == 1 ? t : t / tiles_n;
  const int tn = t - ti.tm * tiles_n;
  ti.m0 = ti.tm * TM;
  ti.n0 = tn * TN;
  const int chunk_r = ((splitR > 1 ? (R + splitR - 1) / splitR : R) + TK - 1) / TK * TK;
  ti.r_begin = split * chunk_r;
  ti.r_end = min(R, ti.r_begin + chunk_r);
  ti.nchunks = ti.r_end > ti.r_begin ? (ti.r_end - ti.r_begin + TK - 1) / TK : 0;
  ti.un = min(TN, ((d.N - ti.n0) + 15) / 16 * 16);   // MMA N for this tile (multiple of 16; the wgmma issues 32 or 64)
  return ti;
}

// enc: the encoder forward's instantiation (planes only, encoder.cu): adds the GG_EPI_BIAS_LRELU epilogue and lets a descriptor
// without C write only its BF16 planes (C_hi / C_lo: the next layer's input).
// ae: the auto-encoder training instantiations (register-staged fp32 operands only, autoencoder.cu, GG_ACC64): the
// GG_EPI_BIAS_LRELU epilogue, the LeakyReLU-derivative epilogue GG_EPI_LRELU_GRAD (C = acc * g(mask), g = 1 / alpha / 0 for a
// stored LeakyReLU output > 0 / < 0 / == 0), and GG_EPI_ATOMIC / GG_COLSUM adding each split's fp32 partial sums into DOUBLE
// arrays behind C / colsum with double atomics.  Every other launch runs enc = ae = false, whose code is the engine as it was
// before the flags existed.
template <bool a_rvec, bool b_rvec, bool planes, bool enc = false, bool ae = false>
__global__ void __launch_bounds__(Roles<planes>::NTHREADS, 1) gg_tc_kernel(const __grid_constant__ DescPack pk, int x3) {
  constexpr int NPROD = Roles<planes>::NPROD, MMA_WARP = Roles<planes>::MMA_WARP, NEPI = Roles<planes>::NEPI;
  constexpr int EPI_COLS = Roles<planes>::EPI_COLS;
  constexpr int MASKF = ae ? (GG_EPI_MASK | GG_EPI_LRELU_GRAD) : GG_EPI_MASK;   // flags that read mask[kM[m] + kN[n]]
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_full[STAGES], bar_empty[STAGES];
  __shared__ int s_cn[TN], s_kn[TN];
  __shared__ __align__(16) float s_bias[TN];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&bar_full[s]), NPROD);
      mbar_init(smem_u32(&bar_empty[s]), NEPI / 32);     // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const uint32_t ring = (smem_u32(smem_raw) + 1023u) & ~1023u;
  pdl_trigger();      // the next kernel on the stream may begin its own prologue now
  pdl_wait();         // everything above overlapped the predecessor; its results are visible from here on
  // Tile schedule: round-robin over the grid
  const int t_begin = blockIdx.x, t_end = pk.total_tiles, t_step = gridDim.x;

  if (planes && warp < MMA_WARP) {
    // =========================================================================== producers (BF16 planes, cp.async)
    // Operands are already split into BF16 hi/lo planes in HBM: every 16-byte chunk of a wgmma tile is one
    // cp.async straight into its swizzled slot -- no registers, no conversion; the ring depth is the prefetch
    // depth, and the slot's mbarrier is signalled by the copies themselves (cp.async.mbarrier.arrive.noinc).
    const int c8 = tid & 7, q = tid >> 3;      // 16-byte chunk, row group: A rows q + 32 i (i < 4), B rows q + 32 i (i < 2)
    uint32_t gc = 0;
    // per-tile gather state, fetched ONE TILE AHEAD so that the row-offset / table round trips of tile i+1
    // overlap the copies of tile i (the ring keeps running across tile boundaries)
    // qa / ca: this thread's A row group and 16-byte column group.  Default: 8 lanes span one row's 128 bytes
    // (dense rows: one line per row).  GG_A_ROWLANES: 8 lanes span 8 consecutive rows of one column group.
    struct TState { TileInfo ti; int a_off[4]; bool a_ok[4]; int b_off[2]; bool b_ok[2]; int ta[4], tb[4]; int qa, ca; bool valid; };
    auto fetch = [&](int tile) {
      TState t;
      t.valid = tile < t_end;
      if (!t.valid) return t;
      t.ti = tile_info(pk, tile);
      const GemmDesc& d = pk.d[t.ti.p];
      const int dfl = d.flags;
      if (dfl & GG_MN_MAJOR) return t;           // MN-major tiles fetch their (few) offsets in place
      const bool rl = dfl & GG_A_ROWLANES;
      t.qa = rl ? (tid & 7) + 8 * (tid >> 6) : q;
      t.ca = rl ? (tid >> 3) & 7 : c8;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int m = t.ti.m0 + t.qa + 32 * i;
        t.a_ok[i] = m < d.M;
        t.a_off[i] = t.a_ok[i] ? d.aM[m] : 0;
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int nB = t.ti.n0 + q + 32 * i;
        t.b_ok[i] = nB < d.N;
        t.b_off[i] = t.b_ok[i] ? (d.bN_p ? d.bN_p : d.bN)[nB] : 0;
      }
      // r-offset table entries of the first four r-chunks (the ring depth): short tiles (dgrad: 4 chunks) never wait
      // for a table round trip inside the chunk loop; longer ones keep loading four chunks ahead
      const int* tA = d.aR;
      const int* tB = d.bR_p ? d.bR_p : d.bR;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        t.ta[k] = t.tb[k] = 0;
        if (k < t.ti.nchunks) {
          t.ta[k] = tA[t.ti.r_begin + k * TK + t.ca * 8];
          t.tb[k] = tB[t.ti.r_begin + k * TK + c8 * 8];
        }
      }
      return t;
    };
    TState cur = fetch(t_begin);
    int pin_p = -1, pflags = 0;
    const uint16_t* pA_hi = nullptr; const uint16_t* pA_lo = nullptr; const uint16_t* pB_hi = nullptr; const uint16_t* pB_lo = nullptr;
    const int* tabA = nullptr; const int* tabB_k = nullptr; const int* tabB_mn = nullptr;
    for (int tile = t_begin; tile < t_end; tile += t_step) {
      const TState nxt = fetch(tile + t_step);
      const TileInfo ti = cur.ti;
      if (ti.p != pin_p) {
        const GemmDesc& dd = pk.d[ti.p];
        pflags = pin(dd.flags);
        pA_hi = pin(dd.A_hi); pA_lo = pin(dd.A_lo); pB_hi = pin(dd.B_hi); pB_lo = pin(dd.B_lo);
        tabA = pin(dd.aR); tabB_mn = pin(dd.bR); tabB_k = pin(dd.bR_p ? dd.bR_p : dd.bR);
        pin_p = ti.p;
      }
      if (ti.nchunks > 0 && (pflags & GG_MN_MAJOR)) {
        // ---- wgrad: D[k, n] = sum_m act[m -> k] * dZ[m, n]; both operands are contiguous along their M / N
        // index for a fixed reduction index m, so tiles are MN-major: row (r = m) x 16-byte groups along k / n.
        const GemmDesc& d = pk.d[ti.p];
        const bool align4 = pflags & GG_A_ALIGN4;
        const int* const tabB = tabB_mn;
        // 16-byte group c; reduction rows qq and qq + 32.  GG_A_ROWLANES: 8 lanes walk 8 consecutive reduction rows
        // (adjacent output pixels: overlapping image patches, contiguous dZ rows) instead of the 8 groups of one row
        const bool rl = pflags & GG_A_ROWLANES;
        const int c = rl ? (tid >> 3) & 7 : tid & 7;
        const int qq = rl ? (tid & 7) + 8 * (tid >> 6) : q;
        // column-side offsets of this thread's groups (A: k groups c and c + 8; B: n group c) are tile constants
        const int kg0 = ti.m0 + 8 * c, kg1 = ti.m0 + 8 * (c + 8), ng = ti.n0 + 8 * c;
        const bool k0_ok = kg0 < d.M, k1_ok = kg1 < d.M, n_ok = ng < d.N;
        const int ka0 = k0_ok ? d.aM[kg0] : 0, ka1 = k1_ok ? d.aM[kg1] : 0, nb_ = n_ok ? d.bN[ng] : 0;
        for (int ch = 0; ch < ti.nchunks; ++ch, ++gc) {
          const int s = gc % STAGES;
          const uint32_t sA_hi = ring + s * STAGE_BYTES, sA_lo = sA_hi + A_BYTES;
          const uint32_t sB_hi = sA_lo + A_BYTES, sB_lo = sB_hi + B_BYTES;
          int ar[2], br[2];
          bool r_ok[2];
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int r = ti.r_begin + ch * TK + qq + 32 * u;
            r_ok[u] = r < ti.r_end;
            ar[u] = r_ok[u] ? tabA[r] : 0;
            br[u] = r_ok[u] ? tabB[r] : 0;
          }
          if (gc >= STAGES) mbar_wait(smem_u32(&bar_empty[s]), ((gc / STAGES) - 1) & 1);
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int rr = qq + 32 * u;
            const int ki = rr >> 3, kk = rr & 7;
            const uint32_t swz = (uint32_t)((c ^ kk) << 4);
            const uint32_t oA0 = (uint32_t)(ki * 2048 + kk * 128) + swz, oA1 = oA0 + 1024, oB = (uint32_t)(ki * 1024 + kk * 128) + swz;
            const int nb0 = (r_ok[u] && k0_ok) ? 16 : 0, nb1 = (r_ok[u] && k1_ok) ? 16 : 0, nbb = (r_ok[u] && n_ok) ? 16 : 0;
            const size_t e0 = (size_t)(ar[u] + ka0), e1 = (size_t)(ar[u] + ka1), eb = (size_t)(br[u] + nb_);
            if (!align4) {
              cp_async16(sA_hi + oA0, pA_hi + e0, nb0);
              cp_async16(sA_hi + oA1, pA_hi + e1, nb1);
              if (x3) { cp_async16(sA_lo + oA0, pA_lo + e0, nb0); cp_async16(sA_lo + oA1, pA_lo + e1, nb1); }
            } else {
              cp_async8(sA_hi + oA0, pA_hi + e0, nb0 / 2); cp_async8(sA_hi + oA0 + 8, pA_hi + e0 + 4, nb0 / 2);
              cp_async8(sA_hi + oA1, pA_hi + e1, nb1 / 2); cp_async8(sA_hi + oA1 + 8, pA_hi + e1 + 4, nb1 / 2);
              if (x3) {
                cp_async8(sA_lo + oA0, pA_lo + e0, nb0 / 2); cp_async8(sA_lo + oA0 + 8, pA_lo + e0 + 4, nb0 / 2);
                cp_async8(sA_lo + oA1, pA_lo + e1, nb1 / 2); cp_async8(sA_lo + oA1 + 8, pA_lo + e1 + 4, nb1 / 2);
              }
            }
            cp_async16(sB_hi + oB, pB_hi + eb, nbb);
            if (x3) cp_async16(sB_lo + oB, pB_lo + eb, nbb);
          }
          cp_async_arrive_noinc(smem_u32(&bar_full[s]));
        }
      } else if (ti.nchunks > 0) {
        const bool align4 = pflags & GG_A_ALIGN4;
        const int* const tabB = tabB_k;
        int ta0 = cur.ta[0], ta1 = cur.ta[1], ta2 = cur.ta[2], ta3 = cur.ta[3];
        int tb0 = cur.tb[0], tb1 = cur.tb[1], tb2 = cur.tb[2], tb3 = cur.tb[3];
        for (int ch = 0; ch < ti.nchunks; ++ch, ++gc) {
          const int ta = ta0, tb = tb0;
          const int s = gc % STAGES;
          const uint32_t sA_hi = ring + s * STAGE_BYTES, sA_lo = sA_hi + A_BYTES;
          const uint32_t sB_hi = sA_lo + A_BYTES, sB_lo = sB_hi + B_BYTES;
          const int r0 = ti.r_begin + ch * TK + c8 * 8, r0a = ti.r_begin + ch * TK + cur.ca * 8;
          const int nbytes = max(0, min(8, ti.r_end - r0)) * 2, nbytes_a = max(0, min(8, ti.r_end - r0a)) * 2;
          if (gc >= STAGES) mbar_wait(smem_u32(&bar_empty[s]), ((gc / STAGES) - 1) & 1);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const uint32_t o = sw128(cur.qa + 32 * i, cur.ca);
            const int nb = cur.a_ok[i] ? nbytes_a : 0;
            const size_t e = (size_t)(cur.a_off[i] + ta);
            if (!align4) {
              cp_async16(sA_hi + o, pA_hi + e, nb);
              if (x3) cp_async16(sA_lo + o, pA_lo + e, nb);
            } else {
              cp_async8(sA_hi + o, pA_hi + e, min(nb, 8));
              cp_async8(sA_hi + o + 8, pA_hi + e + 4, max(nb - 8, 0));
              if (x3) {
                cp_async8(sA_lo + o, pA_lo + e, min(nb, 8));
                cp_async8(sA_lo + o + 8, pA_lo + e + 4, max(nb - 8, 0));
              }
            }
          }
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const uint32_t o = sw128(q + 32 * i, c8);
            const int nb = cur.b_ok[i] ? nbytes : 0;
            const size_t e = (size_t)(cur.b_off[i] + tb);
            cp_async16(sB_hi + o, pB_hi + e, nb);
            if (x3) cp_async16(sB_lo + o, pB_lo + e, nb);
          }
          cp_async_arrive_noinc(smem_u32(&bar_full[s]));
          ta0 = ta1; ta1 = ta2; ta2 = ta3; tb0 = tb1; tb1 = tb2; tb2 = tb3;
          if (ch + 4 < ti.nchunks) { ta3 = tabA[r0a + 4 * TK]; tb3 = tabB[r0 + 4 * TK]; }
        }
      }
      cur = nxt;
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
  } else if (warp < MMA_WARP) {
    // =========================================================================== producers
    const int c8 = tid & 7;             // 16-byte chunk (8 r values) inside the 64-wide r-chunk
    const int q = tid >> 3;             // 0..63
    // A, r-contiguous: all threads, rows q + 64 i (i < 2).  A, m-contiguous: threads < 256, rows 4 q .. 4 q + 3.
    const bool a_thread = a_rvec ? true : (q < 32);
    // B, n-contiguous: threads 256..383 (qb in 0..15), n = 4 qb .. +3.  B, r-contiguous: all threads, n = q.
    const int qb = b_rvec ? q : q - 32;
    const bool b_thread = b_rvec ? true : (qb >= 0 && qb < TN / 4);
    uint32_t gc = 0;                    // ring chunk counter, continuous across tiles

    for (int tile = t_begin; tile < t_end; tile += t_step) {
      const TileInfo ti = tile_info(pk, tile);
      if (ti.nchunks == 0) continue;
      const GemmDesc& d = pk.d[ti.p];
      const float* __restrict__ A = pin(d.A);
      const float* __restrict__ Bp = pin(d.B);
      const bool do_colsum = (d.flags & GG_COLSUM) && ti.tm == 0 && !b_rvec;
      int a_off[4], b_off[4];
      bool a_ok[4], b_ok[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int m = ti.m0 + (a_rvec ? q + 64 * i : 4 * q + i);
        a_ok[i] = a_thread && m < d.M && (a_rvec ? i < 2 : true);
        a_off[i] = a_ok[i] ? d.aM[m] : 0;
        const int n = ti.n0 + (b_rvec ? qb : 4 * qb + i);
        b_ok[i] = b_thread && n < d.N && (b_rvec ? i < 1 : true);
        b_off[i] = b_ok[i] ? d.bN[n] : 0;
      }
      float4 csum = make_float4(0, 0, 0, 0);

      // r-offset table entries of the thread's 8 r values: loaded one chunk ahead so that the operand
      // loads of a chunk are a single batch of independent LDG.128 (one round trip).
      // r-contiguous operands need entries 0 and 4 only; block (m-/n-contiguous) operands need all 8.
      const int* __restrict__ tabA = pin(d.aR);
      const int* __restrict__ tabB = pin(d.bR);
      const bool blk_is_B = !a_rvec && !a_thread;           // wgrad: this thread gathers the B operand
      const int* __restrict__ tabBlk = a_rvec ? tabB : (blk_is_B ? tabB : tabA);
      int t2a[2] = {0, 0}, t2b[2] = {0, 0};                 // r-contiguous A / B
      int t8[8] = {0, 0, 0, 0, 0, 0, 0, 0};                 // block operand (A m-contig, or B n-contig)
      const bool need_blk = a_rvec ? (!b_rvec && b_thread) : (a_thread || b_thread);
      auto load_tabs = [&](int r, int n_valid, int (&o2a)[2], int (&o2b)[2], int (&o8)[8]) {
        if (n_valid == 8) {
          if (a_rvec) { o2a[0] = tabA[r]; o2a[1] = tabA[r + 4]; }
          if (b_rvec) { o2b[0] = tabB[r]; o2b[1] = tabB[r + 4]; }
          if (need_blk) {
            const int4 u = *reinterpret_cast<const int4*>(tabBlk + r), w = *reinterpret_cast<const int4*>(tabBlk + r + 4);
            o8[0] = u.x; o8[1] = u.y; o8[2] = u.z; o8[3] = u.w; o8[4] = w.x; o8[5] = w.y; o8[6] = w.z; o8[7] = w.w;
          }
        }
      };
      {
        const int r00 = ti.r_begin + c8 * 8;
        load_tabs(r00, min(8, ti.r_end - r00), t2a, t2b, t8);
      }

      for (int ch = 0; ch < ti.nchunks; ++ch, ++gc) {
        const int s = gc % STAGES;
        const uint32_t sA_hi = ring + s * STAGE_BYTES, sA_lo = sA_hi + A_BYTES;
        const uint32_t sB_hi = sA_lo + A_BYTES, sB_lo = sB_hi + B_BYTES;
        const int r0 = ti.r_begin + ch * TK + c8 * 8;
        const int nr = min(8, ti.r_end - r0);            // valid r values (<= 0: none)
        // ---------------------------------------------------------------- issue every global load first
        float xa[4][8];     // rvec: [unit i][r j] (i < 2);  mvec: [m i][r j]  (wgrad: B-threads reuse it)
        float xb[4][8];     // rvec: [0][r j];                nvec: [n i][r j]
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) xa[i][j] = xb[i][j] = 0.f;
        if (nr == 8) {
          // ---- fast path: full 8-wide r group, straight-line independent loads
          if (a_rvec) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              if (a_ok[i]) {
                const float4 v = ldg4(A + a_off[i] + t2a[0]), w = ldg4(A + a_off[i] + t2a[1]);
                xa[i][0] = v.x; xa[i][1] = v.y; xa[i][2] = v.z; xa[i][3] = v.w;
                xa[i][4] = w.x; xa[i][5] = w.y; xa[i][6] = w.z; xa[i][7] = w.w;
              }
            }
          }
          if (b_rvec) {
            if (b_ok[0]) {
              const float4 v = ldg4(Bp + b_off[0] + t2b[0]), w = ldg4(Bp + b_off[0] + t2b[1]);
              xb[0][0] = v.x; xb[0][1] = v.y; xb[0][2] = v.z; xb[0][3] = v.w;
              xb[0][4] = w.x; xb[0][5] = w.y; xb[0][6] = w.z; xb[0][7] = w.w;
            }
          }
          if (need_blk) {
            float (&xq)[4][8] = a_rvec ? xb : xa;
            const float* __restrict__ base = (a_rvec || blk_is_B) ? Bp : A;
            const int (&off)[4] = (a_rvec || blk_is_B) ? b_off : a_off;
            const bool (&ok)[4] = (a_rvec || blk_is_B) ? b_ok : a_ok;
            if (ok[3]) {
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const float4 v = ldg4(base + off[0] + t8[j]);
                xq[0][j] = v.x; xq[1][j] = v.y; xq[2][j] = v.z; xq[3][j] = v.w;
              }
            } else {
#pragma unroll
              for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int i = 0; i < 4; ++i)
                  if (ok[i]) xq[i][j] = base[off[i] + t8[j]];
            }
          }
        } else if (nr > 0) {
          // ---- slow path: ragged tail of the r range
          if (a_rvec) {
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
              for (int j = 0; j < 8; ++j)
                if (a_ok[i] && j < nr) xa[i][j] = A[a_off[i] + tabA[r0 + j]];
          } else if (a_thread) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
              for (int i = 0; i < 4; ++i)
                if (a_ok[i] && j < nr) xa[i][j] = A[a_off[i] + tabA[r0 + j]];
          }
          if (b_rvec) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
              if (b_ok[0] && j < nr) xb[0][j] = Bp[b_off[0] + tabB[r0 + j]];
          } else if (b_thread) {
            float (&xq)[4][8] = a_rvec ? xb : xa;
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
              for (int i = 0; i < 4; ++i)
                if (b_ok[i] && j < nr) xq[i][j] = Bp[b_off[i] + tabB[r0 + j]];
          }
        }
        if (do_colsum && b_thread) {
          float (&xq)[4][8] = a_rvec ? xb : xa;
#pragma unroll
          for (int j = 0; j < 8; ++j) { csum.x += xq[0][j]; csum.y += xq[1][j]; csum.z += xq[2][j]; csum.w += xq[3][j]; }
        }
        // table entries of the next chunk (in flight during the wait + split + store below)
        if (ch + 1 < ti.nchunks) {
          const int r1 = r0 + TK;
          load_tabs(r1, min(8, ti.r_end - r1), t2a, t2b, t8);
        }
        // ---------------------------------------------------------------- ring slot free?  then split + store
        if (gc >= STAGES) mbar_wait(smem_u32(&bar_empty[s]), ((gc / STAGES) - 1) & 1);
        if (a_thread) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            if (a_rvec && i >= 2) break;
            uint4 hi, lo;
            split8(xa[i], hi, lo);
            const uint32_t o = sw128(a_rvec ? q + 64 * i : 4 * q + i, c8);
            st_shared16(sA_hi + o, hi);
            if (x3) st_shared16(sA_lo + o, lo);
          }
        }
        if (b_thread) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            if (b_rvec && i >= 1) break;
            uint4 hi, lo;
            split8((a_rvec || b_rvec) ? xb[i] : xa[i], hi, lo);
            const uint32_t o = sw128(b_rvec ? qb : 4 * qb + i, c8);
            st_shared16(sB_hi + o, hi);
            if (x3) st_shared16(sB_lo + o, lo);
          }
        }
        fence_proxy_async();                 // generic-proxy smem writes -> visible to the tensor-core (async) proxy
        mbar_arrive(smem_u32(&bar_full[s]));
      }
      if (do_colsum && b_thread) {           // bias gradients: column sums of the B operand rows of this r-range
        const int nb = ti.n0 + 4 * qb;
        if (ae) {
          double* cs = reinterpret_cast<double*>(d.colsum);
          if (nb + 0 < d.N) atomicAdd(cs + nb + 0, (double)csum.x);
          if (nb + 1 < d.N) atomicAdd(cs + nb + 1, (double)csum.y);
          if (nb + 2 < d.N) atomicAdd(cs + nb + 2, (double)csum.z);
          if (nb + 3 < d.N) atomicAdd(cs + nb + 3, (double)csum.w);
        } else {
          if (nb + 0 < d.N) atomicAdd(d.colsum + nb + 0, csum.x);
          if (nb + 1 < d.N) atomicAdd(d.colsum + nb + 1, csum.y);
          if (nb + 2 < d.N) atomicAdd(d.colsum + nb + 2, csum.z);
          if (nb + 3 < d.N) atomicAdd(d.colsum + nb + 3, csum.w);
        }
      }
    }
  } else {
    // =========================================================================== consumers: MMA + epilogue
    // Mainloop: every consumer warpgroup issues the wgmmas of its m64 blocks for each ring chunk, waits for them and frees the
    // slot (one arrival per warp).  Epilogue: the accumulators go to the shared accumulator tile, after which each warp owns 32
    // rows (its lane quarter) x EPI_COLS columns.  Column-side tables (cN, kN, bias) of the tile are staged in shared memory
    // BEFORE the mainloop.  Phase A: accumulator tile -> (+bias, ReLU) -> the warp's private fp32 staging rows.  Phase B: staging rows -> (ReLU mask) -> global, fully coalesced: LPR lanes cover one row's
    // contiguous run (fp32 float4 + BF16 hi/lo uint2), 32/LPR rows per instruction, loads batched ahead of stores.
    // Fast-path contract (GG_CN_AFFINE4, verified on the host): inside every aligned group of 4 columns cN / kN are
    // contiguous and the output offset is 16-byte aligned.
    const int ew = warp - MMA_WARP;                // consumer warp index
    const int lq = warp & 3;                       // row quarter of the tile this warp stores
    const int et = tid - MMA_WARP * 32;            // 0..NEPI-1
    constexpr int MB = Roles<planes>::MB;
    const int m_first = (ew >> 2) * MB;            // first m64 block of this warpgroup
    const uint32_t accs = ring + STAGES * STAGE_BYTES + STG_BYTES;
    uint32_t gcm = 0;                              // ring chunk counter, continuous across tiles
    int pinned_p = -1, dflags = 0, dN = 0;
    float* dC = nullptr; uint16_t* dChi = nullptr; uint16_t* dClo = nullptr; const float* dmask = nullptr;
    float dalpha = 0.f;                            // enc, ae: LeakyReLU slope
    const uint32_t stg = ring + STAGES * STAGE_BYTES + (uint32_t)ew * (32 * EPI_COLS * 4);
    int staged_n0 = -1, st_col = -2;               // which (column tables, column block) the staged copies belong to
    // Everything a tile's epilogue needs from global memory besides the mask -- tile coordinates, this lane's row
    // offsets (cM / kM), this thread's column-table entry (cN / kN / bias) -- is fetched ONE TILE AHEAD and only
    // consumed after the current tile's work, so none of those round trips sits on the per-tile critical path.
    // No arithmetic touches a freshly loaded value inside prefetch() (a dependent instruction would stall there).
    struct ENext { TileInfo ti; int cm, km; bool ok, km_same, valid; int t_cn, t_kn; float t_bias; bool kn_same; int col_id; };
    auto prefetch = [&](int tile) {
      ENext e;
      e.valid = tile < t_end;
      e.cm = e.km = 0; e.ok = false; e.km_same = true; e.t_cn = e.t_kn = 0; e.t_bias = 0.f; e.kn_same = true;
      e.col_id = -1;
      if (!e.valid) return e;
      e.ti = tile_info(pk, tile);
      if (e.ti.nchunks == 0) return e;
      const GemmDesc& d2 = pk.d[e.ti.p];
      const int fl = d2.flags;
      // identity of the column tables (host-assigned: same cN / kN / bias / N -> same id): problems that share them
      // (the parity-class dgrads of a layer, both nets) do not re-stage -- and so skip the named-barrier pair -- when a
      // CTA's consecutive tiles hop between them
      e.col_id = d2.col_id;
      const int m2 = e.ti.m0 + lq * 32 + lane;
      e.ok = m2 < d2.M;
      if (e.ok) e.cm = d2.cM[m2];
      const int* kMp = d2.kM;
      e.km_same = !((fl & MASKF) && kMp);
      if (e.ok && !e.km_same) e.km = kMp[m2];
      if (et < TN) {
        const int n = e.ti.n0 + et;
        if (n < d2.N) {
          e.t_cn = d2.cN[n];
          const int* kNp = d2.kN;
          e.kn_same = kNp == nullptr;
          if (kNp) e.t_kn = kNp[n];
        }
      } else if (et < 2 * TN) {
        const int n = e.ti.n0 + et - TN;
        if ((fl & (enc || ae ? GG_EPI_BIAS_RELU | GG_EPI_BIAS_LRELU : GG_EPI_BIAS_RELU)) && n < d2.N) e.t_bias = d2.bias[n];
      }
      return e;
    };
    ENext nxt = prefetch(t_begin);
    for (int tile = t_begin; tile < t_end; tile += t_step) {
      const ENext cur = nxt;
      nxt = prefetch(tile + t_step);
      const TileInfo ti = cur.ti;
      if (ti.nchunks == 0) continue;
      const int cm = cur.cm, km = cur.km_same ? cur.cm : cur.km;
      const bool m_ok = cur.ok;
      const GemmDesc& d = pk.d[ti.p];
      if (cur.col_id != st_col || ti.n0 != staged_n0) {   // block-uniform: every epilogue warp walks the same tiles
        asm volatile("bar.sync 2, %0;" ::"n"(NEPI));  // previous readers of the staged tables are done
        if (et < TN) {
          s_cn[et] = cur.t_cn;
          s_kn[et] = cur.kn_same ? cur.t_cn : cur.t_kn;
        } else if (et < 2 * TN) {
          s_bias[et - TN] = cur.t_bias;
        }
        asm volatile("bar.sync 2, %0;" ::"n"(NEPI));
        st_col = cur.col_id; staged_n0 = ti.n0;
      }
      if (ti.p != pinned_p) {      // register copies of everything the store loops need from the descriptor
        dflags = pin(d.flags); dN = pin(d.N);
        dC = pin(d.C); dChi = pin(d.C_hi); dClo = pin(d.C_lo); dmask = pin(d.mask);
        if (enc || ae) dalpha = d.alpha;
        pinned_p = ti.p;
      }
      // column split between the two warps of a row quarter (8 epilogue warps, planes mode): 32 + 32 columns,
      // or 16 + 16 when the tile is at most 32 wide (conv1 fwd / wgrad, conv2 dgrad) so that no warp idles
      const int ecols = (NEPI == 256 && ti.un <= 32) ? 16 : EPI_COLS;
      const int col0 = (ew >> 2) * ecols;            // first accumulator column of this warp
      const int lpr_log = ecols == 16 ? 2 : (EPI_COLS == 64 ? 4 : 3), LPR = 1 << lpr_log, RPI = 32 >> lpr_log;
      const bool fastp = (dflags & GG_CN_AFFINE4) && (ti.n0 + ti.un <= dN);
      const int ncols_w = max(0, min(ecols, ti.un - col0));        // warp-uniform, multiple of 16
      // ReLU-mask values of the first store batch: their addresses depend only on the tables, so the loads are issued
      // before the accumulator is even waited for and have landed by the time phase B needs them
      float4 mk0[4];
      const int pc = lane & (LPR - 1), psub = lane >> lpr_log;
      const bool pact = pc < (ncols_w >> 2);
      const bool early_mask = planes && fastp && (dflags & GG_EPI_MASK) && ncols_w > 0;   // (register budget: planes kernel only)
      {
        const int kn = (early_mask && pact) ? s_kn[col0 + 4 * pc] : 0;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int row = RPI * u + psub;
          const int km_r = __shfl_sync(0xffffffffu, km, row & 31);
          const bool ok_r = __shfl_sync(0xffffffffu, (int)m_ok, row & 31) != 0;
          mk0[u] = make_float4(1, 1, 1, 1);
          if (early_mask && pact && ok_r && row < 32) mk0[u] = ldg4(dmask + km_r + kn);
        }
      }
      {
        float acc[MB][32];
#pragma unroll
        for (int mb = 0; mb < MB; ++mb)
#pragma unroll
          for (int j = 0; j < 32; ++j) acc[mb][j] = 0.f;
        const bool mnm = planes && (dflags & GG_MN_MAJOR);
        for (int ch = 0; ch < ti.nchunks; ++ch, ++gcm) {
          const int s = gcm % STAGES;
          mbar_wait(smem_u32(&bar_full[s]), (gcm / STAGES) & 1);
          if (planes) fence_proxy_async();       // cp.async (generic proxy) writes -> tensor-core (async proxy) reads
          const uint32_t sA_hi = ring + s * STAGE_BYTES, sA_lo = sA_hi + A_BYTES;
          const uint32_t sB_hi = sA_lo + A_BYTES, sB_lo = sB_hi + B_BYTES;
          wg_arrive();
          if (mnm) mma_chunk<64, 1, MB>(acc, sA_hi, sA_lo, sB_hi, sB_lo, m_first, x3);
          else if (ti.un <= 32) mma_chunk<32, 0, MB>(acc, sA_hi, sA_lo, sB_hi, sB_lo, m_first, x3);
          else mma_chunk<64, 0, MB>(acc, sA_hi, sA_lo, sB_hi, sB_lo, m_first, x3);
          wg_commit();
          wg_wait<0>();
          __syncwarp();
          if (lane == 0) mbar_arrive(smem_u32(&bar_empty[s]));     // the ring slot may be refilled
        }
        // accumulator fragments -> the shared accumulator tile (every consumer has read the previous tile's rows)
        asm volatile("bar.sync 3, %0;" ::"n"(NEPI));
#pragma unroll
        for (int mb = 0; mb < MB; ++mb)
#pragma unroll
          for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = 64 * (m_first + mb) + 16 * (ew & 3) + (lane >> 2) + 8 * h;
              const int chunk = 2 * j + ((lane & 3) >> 1);
              const uint32_t a = accs + (uint32_t)row * 256u + (uint32_t)((chunk ^ (row & 7)) << 4) + (uint32_t)((lane & 1) * 8);
              asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(a), "f"(acc[mb][4 * j + 2 * h]), "f"(acc[mb][4 * j + 2 * h + 1]) : "memory");
            }
        asm volatile("bar.sync 3, %0;" ::"n"(NEPI));
      }
#pragma unroll 1
      for (int cb = col0; cb < col0 + ncols_w; cb += 16) {
        uint32_t v[16];
        {
          const int row = lq * 32 + lane;
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            const uint32_t a = accs + (uint32_t)row * 256u + (uint32_t)((((cb >> 2) + g) ^ (row & 7)) << 4);
            asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v[4 * g]), "=r"(v[4 * g + 1]), "=r"(v[4 * g + 2]), "=r"(v[4 * g + 3]) : "r"(a));
          }
        }
        if (fastp) {
          // phase A: accumulator row -> (+bias, ReLU) -> this warp's staging rows (16-byte chunks XOR-swizzled by row)
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            float4 o = make_float4(__uint_as_float(v[4 * g]), __uint_as_float(v[4 * g + 1]), __uint_as_float(v[4 * g + 2]),
                                   __uint_as_float(v[4 * g + 3]));
            if (dflags & GG_EPI_BIAS_RELU) {
              const float4 bb = *reinterpret_cast<const float4*>(&s_bias[cb + 4 * g]);
              o.x = fmaxf(o.x + bb.x, 0.f); o.y = fmaxf(o.y + bb.y, 0.f); o.z = fmaxf(o.z + bb.z, 0.f); o.w = fmaxf(o.w + bb.w, 0.f);
            }
            if ((enc || ae) && (dflags & GG_EPI_BIAS_LRELU)) {     // gg_simt's order: v + bias, then v > 0 ? v : alpha * v
              const float4 bb = *reinterpret_cast<const float4*>(&s_bias[cb + 4 * g]);
              o.x += bb.x; o.y += bb.y; o.z += bb.z; o.w += bb.w;
              o.x = o.x > 0.f ? o.x : dalpha * o.x; o.y = o.y > 0.f ? o.y : dalpha * o.y;
              o.z = o.z > 0.f ? o.z : dalpha * o.z; o.w = o.w > 0.f ? o.w : dalpha * o.w;
            }
            const int c = ((cb - col0) >> 2) + g;
            const uint32_t a = stg + (uint32_t)lane * (EPI_COLS * 4) + (uint32_t)((c ^ (lane & 7)) << 4);
            asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(a), "f"(o.x), "f"(o.y), "f"(o.z), "f"(o.w) : "memory");
          }
        } else if (m_ok) {
          const int nb0 = ti.n0 + cb;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int n = nb0 + j;
            if (n >= dN) break;
            float o = __uint_as_float(v[j]);
            const int cnj = s_cn[cb + j];
            if (dflags & GG_EPI_BIAS_RELU) o = fmaxf(o + s_bias[cb + j], 0.f);
            if ((enc || ae) && (dflags & GG_EPI_BIAS_LRELU)) { o += s_bias[cb + j]; o = o > 0.f ? o : dalpha * o; }
            if (dflags & GG_EPI_MASK) o = dmask[km + s_kn[cb + j]] > 0.f ? o : 0.f;
            if (ae && (dflags & GG_EPI_LRELU_GRAD)) {
              const float mv = dmask[km + s_kn[cb + j]];
              o = mv > 0.f ? o : (mv < 0.f ? o * dalpha : 0.f);
            }
            if (ae && (dflags & GG_EPI_ATOMIC)) atomicAdd(reinterpret_cast<double*>(dC) + cm + cnj, (double)o);
            else if (dflags & GG_EPI_ATOMIC) atomicAdd(dC + cm + cnj, o);
            else if (!enc || dC) dC[cm + cnj] = o;
            if (dChi) {
              const __nv_bfloat16 h = __float2bfloat16_rn(o);
              dChi[cm + cnj] = __bfloat16_as_ushort(h);
              dClo[cm + cnj] = __bfloat16_as_ushort(__float2bfloat16_rn(o - __bfloat162float(h)));
            }
          }
        }
      }
      if (fastp && ncols_w > 0) {
        __syncwarp();
        const int c = lane & (LPR - 1), sub = lane >> lpr_log;
        const bool act = c < (ncols_w >> 2);
        const int cn = act ? s_cn[col0 + 4 * c] : 0, kn = act ? s_kn[col0 + 4 * c] : 0;
#pragma unroll 1
        for (int rr0 = 0; rr0 < 32; rr0 += 4 * RPI) {
          // batch of 4 row groups: every shared / global LOAD first, then math + stores (the compiler cannot hoist
          // loads over stores, so the batching is explicit)
          float4 o[4], mk[4];
          int cmr[4];
          bool okr[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int row = rr0 + RPI * u + sub;
            cmr[u] = __shfl_sync(0xffffffffu, cm, row);
            const int km_r = __shfl_sync(0xffffffffu, km, row);
            okr[u] = (__shfl_sync(0xffffffffu, (int)m_ok, row) != 0) && act;
            o[u] = make_float4(0, 0, 0, 0);
            mk[u] = make_float4(1, 1, 1, 1);
            if (okr[u]) {
              const uint32_t a = stg + (uint32_t)row * (EPI_COLS * 4) + (uint32_t)((c ^ (row & 7)) << 4);
              asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(o[u].x), "=f"(o[u].y), "=f"(o[u].z), "=f"(o[u].w) : "r"(a));
              if (dflags & MASKF) mk[u] = (planes && rr0 == 0) ? mk0[u] : ldg4(dmask + km_r + kn);
            }
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            if (!okr[u]) continue;
            float4 v4 = o[u];
            if (ae && (dflags & GG_EPI_LRELU_GRAD)) {
              v4.x = mk[u].x > 0.f ? v4.x : (mk[u].x < 0.f ? v4.x * dalpha : 0.f);
              v4.y = mk[u].y > 0.f ? v4.y : (mk[u].y < 0.f ? v4.y * dalpha : 0.f);
              v4.z = mk[u].z > 0.f ? v4.z : (mk[u].z < 0.f ? v4.z * dalpha : 0.f);
              v4.w = mk[u].w > 0.f ? v4.w : (mk[u].w < 0.f ? v4.w * dalpha : 0.f);
            } else {
              v4.x = mk[u].x > 0.f ? v4.x : 0.f; v4.y = mk[u].y > 0.f ? v4.y : 0.f;
              v4.z = mk[u].z > 0.f ? v4.z : 0.f; v4.w = mk[u].w > 0.f ? v4.w : 0.f;
            }
            if (ae && (dflags & GG_EPI_ATOMIC)) {
              double* cp = reinterpret_cast<double*>(dC) + cmr[u] + cn;
              atomicAdd(cp + 0, (double)v4.x); atomicAdd(cp + 1, (double)v4.y); atomicAdd(cp + 2, (double)v4.z);
              atomicAdd(cp + 3, (double)v4.w);
            } else if (dflags & GG_EPI_ATOMIC) {
              float* cp = dC + cmr[u] + cn;
              atomicAdd(cp + 0, v4.x); atomicAdd(cp + 1, v4.y); atomicAdd(cp + 2, v4.z); atomicAdd(cp + 3, v4.w);
            } else if (!enc || dC) {
              *reinterpret_cast<float4*>(dC + cmr[u] + cn) = v4;
            }
            if (dChi) {
              const float x[8] = {v4.x, v4.y, v4.z, v4.w, 0.f, 0.f, 0.f, 0.f};
              uint4 hi, lo;
              split8(x, hi, lo);
              *reinterpret_cast<uint2*>(dChi + cmr[u] + cn) = make_uint2(hi.x, hi.y);
              *reinterpret_cast<uint2*>(dClo + cmr[u] + cn) = make_uint2(lo.x, lo.y);
            }
          }
        }
        __syncwarp();      // staging rows are reused by the next tile
      }
    }
  }
}

template <bool AR, bool BR, bool PL, bool ENC = false, bool AE = false>
cudaError_t set_smem_attr() {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gg_tc_kernel<AR, BR, PL, ENC, AE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  return cudaSuccess;
}

template <bool AR, bool BR, bool PL, bool ENC = false, bool AE = false>
cudaError_t launch_mode(const DescPack& pk, int x3, int num_sms, cudaStream_t s) {
  if (cudaError_t e = set_smem_attr<AR, BR, PL, ENC, AE>()) return e;
  const int grid = pk.total_tiles < num_sms ? pk.total_tiles : num_sms;
  return launch_pdl(gg_tc_kernel<AR, BR, PL, ENC, AE>, dim3(grid), dim3(Roles<PL>::NTHREADS), SMEM_BYTES, s, pdl_enabled(), pk, x3);
}
}  // namespace

int gg_tc_smem_bytes() { return SMEM_BYTES; }

cudaError_t gg_tc_acc64_init() {
  if (cudaError_t e = set_smem_attr<true, false, false, false, true>()) return e;
  if (cudaError_t e = set_smem_attr<true, true, false, false, true>()) return e;
  return set_smem_attr<false, false, false, false, true>();
}

// All problems of one launch share the operand-contiguity mode (flags & (GG_A_RVEC | GG_B_RVEC)).  GG_PLANES | GG_EPI_BIAS_LRELU
// selects the encoder forward's instantiation, GG_ACC64 the auto-encoder training's (A r-contiguous, or both operands
// m- / n-contiguous: the weight gradients).
// host_descs: the group's descriptors (at most GG_TC_MAX_DESCS), passed as a __grid_constant__ pack.
cudaError_t gg_tc_launch(const GemmDesc* host_descs, int ndesc, int total_tiles, int mode_flags, int x3, int num_sms, cudaStream_t s) {
  if (total_tiles <= 0) return cudaSuccess;
  if (ndesc > GG_TC_MAX_DESCS) return cudaErrorInvalidValue;
  DescPack pk;
  for (int i = 0; i < ndesc; ++i) pk.d[i] = host_descs[i];
  pk.n = ndesc;
  pk.total_tiles = total_tiles;
  const bool ar = mode_flags & GG_A_RVEC, br = mode_flags & GG_B_RVEC;
  if ((mode_flags & GG_PLANES) && (mode_flags & GG_EPI_BIAS_LRELU)) return launch_mode<true, true, true, true>(pk, x3, num_sms, s);
  if (mode_flags & GG_ACC64) {
    if (ar && br) return launch_mode<true, true, false, false, true>(pk, x3, num_sms, s);
    if (ar) return launch_mode<true, false, false, false, true>(pk, x3, num_sms, s);
    if (!br) return launch_mode<false, false, false, false, true>(pk, x3, num_sms, s);
    return cudaErrorInvalidValue;
  }
  if (mode_flags & GG_PLANES) return launch_mode<true, true, true>(pk, x3, num_sms, s);
  if (ar && br) return launch_mode<true, true, false>(pk, x3, num_sms, s);
  if (ar) return launch_mode<true, false, false>(pk, x3, num_sms, s);
  if (br) return launch_mode<false, true, false>(pk, x3, num_sms, s);
  return launch_mode<false, false, false>(pk, x3, num_sms, s);
}

}  // namespace b2g
