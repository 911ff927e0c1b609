// TMA-fed wgmma contraction engine (sm_90a).  See cg.cuh for the problem description.
//
// Persistent, warp-specialised kernel, one CTA per SM, grid = min(#tiles, #SMs):
//   warps 0..7  : two MMA warpgroups.  Warpgroup w issues wgmma.mma_async for rows [64w, 64w + 64) of the 128-row tile
//                 (BF16 planes from the swizzled ring, fp32 accumulators in registers).  Precision modes per problem: 1 product
//                 (hi*hi), 3 products (2-plane split) or 6 products (3-plane split hi/mid/lo: everything down to 2^-24), one
//                 MMA per product into the accumulator of its order (see mma_chunk), one K-chunk of them in flight while the
//                 next chunk is awaited.  After the last K-chunk an ACT / DGRAD tile's sums go to the shared-memory handoff
//                 buffer (acc_full / acc_empty barriers) and the warps start the next tile; a RAW / WGRAD tile is finished in
//                 place: its columns pass, 16 at a time, through a small staging block so that every lane holds one output row,
//                 then the fp32 stores or red.adds;
//   warps 8..11 : the epilogue warpgroup.  Lane l of warp e reads row 32e + l of a handed-off tile (all its columns), then
//                 bias/ReLU or the ReLU mask (+ the bias-gradient column sums), the split into BF16 planes and their 16-byte
//                 vector stores (transposed inside lane quads so that each instruction writes whole 64-byte row segments), the
//                 split-K finalisation and the dependency arrivals -- while the MMA warps run the next tile's mainloop;
//   warps 12..13: TMA producers (whole warps, converged; one elected lane issues).  The cp.async.bulk.tensor boxes of a K-chunk
//                 (operands x planes) are dealt round-robin to the two warps; warp 12 posts the chunk's expect_tx.
//   warps 14..15: complete the producer warpgroup for setmaxnreg and exit.
#include <cuda_bf16.h>

#include <cstdio>
#include <cstdlib>

#include "cg.cuh"
#include "common.cuh"
#include "wgmma.cuh"

namespace b2g {
namespace {

// warps 0..7: MMA warpgroups, warps 8..11: epilogue warpgroup, warps 12..15: producer warpgroup, of which warps 12..13 issue the
// TMA loads and warps 14..15 only hand their registers over (setmaxnreg acts on whole warpgroups)
constexpr int NMMA_WARPS = 8, NEPI_WARPS = CG_EPI_WARPS, NPROD_WARPS = 2;
constexpr int EPI_WARP0 = NMMA_WARPS, PROD_WARP0 = NMMA_WARPS + NEPI_WARPS;
static_assert(NEPI_WARPS == 4, "the epilogue is one warpgroup: one row of the 128-row tile per lane");
constexpr int NTHREADS = 32 * (PROD_WARP0 + 4);
// registers per thread after setmaxnreg: 2 x MMA + EPI + PROD <= 512 per SM sub-partition lane (each holds two MMA warps, one
// epilogue warp and one producer warp), i.e. the whole 64K register file.  The MMA warps hold up to 128 accumulator registers
// across a mainloop in which one chunk's wgmmas are always in flight.
constexpr int MMA_REGS = 168, EPI_REGS = 152, PROD_REGS = 24;
static_assert(2 * MMA_REGS + EPI_REGS + PROD_REGS <= 512, "register file");
constexpr int STG_BYTES = 2 * 64 * 16 * 4;    // in-place epilogue staging: per warpgroup 64 rows x 16 fp32 columns (rows of 64 B)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "CG_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra CG_DONE;\n\t"
      "bra CG_WAIT;\n\t"
      "CG_DONE:\n\t"
      "}" ::"r"(bar), "r"(parity)
      : "memory");
}
// one lane of a CONVERGED warp.  The producer warps run their loops with all 32 lanes so that every address and coordinate
// is warp-uniform and can live in the uniform registers the TMA instruction reads; a role entered by one lane only
// (if (lane == 0) {...}) lets the compiler wrap each such instruction in a value-serialisation loop.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(pred));
  return pred != 0;
}
// shared-memory matrix descriptor: the problem's constant bits (cg_desc_bits: swizzle span, LBO, SBO) | the start address
__device__ __forceinline__ uint64_t desc_at(uint64_t bits, uint32_t saddr) { return bits | (uint64_t)((saddr & 0x3FFFFu) >> 4); }

__device__ __forceinline__ void tma_load(uint32_t dst, const CUtensorMap* map, uint32_t bar, int rank, const int (&c)[5]) {
  switch (rank) {
    case 2:
      asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst), "l"(map),
                   "r"(bar), "r"(c[0]), "r"(c[1])
                   : "memory");
      break;
    case 3:
      asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
                   "l"(map), "r"(bar), "r"(c[0]), "r"(c[1]), "r"(c[2])
                   : "memory");
      break;
    case 4:
      asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
                   "l"(map), "r"(bar), "r"(c[0]), "r"(c[1]), "r"(c[2]), "r"(c[3])
                   : "memory");
      break;
    default:
      asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(
                       dst),
                   "l"(map), "r"(bar), "r"(c[0]), "r"(c[1]), "r"(c[2]), "r"(c[3]), "r"(c[4])
                   : "memory");
      break;
  }
}

// The problem list lives in the kernel-parameter constant bank: every role re-reads descriptor fields per tile, and a
// constant-cache hit costs far less than the dependent L2 round trip per field group of a descriptor in global memory.
struct CgPack { CgProblem p[CG_MAX_PROBLEMS]; };
struct Tile { int p, tm, tn, c_begin, c_end; };
// Tile walker: a CTA's tiles increase monotonically, so the problem index only moves forward and the tile-grid fields of
// the current problem stay in registers (re-read from the constant bank only when the problem changes).
struct Walker {
  int p = -1, next_start = 0, tile_start = 0, tiles_n = 1, per = 1, splits = 1, chunks = 0, cps = 0;
  __device__ __forceinline__ bool advance(const CgProblem* __restrict__ probs, int nprob, int tile) {   // true: problem changed
    bool changed = false;
    while (p < 0 || (p + 1 < nprob && tile >= next_start)) {
      ++p;
      const CgProblem& P = probs[p];
      tile_start = P.tile_start; tiles_n = P.tiles_n; per = P.tiles_m * P.tiles_n; splits = P.splits; chunks = P.chunks;
      cps = (chunks + splits - 1) / splits;
      next_start = p + 1 < nprob ? probs[p + 1].tile_start : 0x7fffffff;
      changed = true;
    }
    return changed;
  }
  __device__ __forceinline__ Tile tile(int t_abs) const {
    int t = t_abs - tile_start, split = 0;
    if (splits > 1) { split = t / per; t -= split * per; }
    Tile ti;
    ti.p = p;
    ti.tm = tiles_n == 1 ? t : t / tiles_n;
    ti.tn = t - ti.tm * tiles_n;
    ti.c_begin = split * cps;
    ti.c_end = min(chunks, ti.c_begin + cps);
    return ti;
  }
};

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {    // lo -> bits [0,16)
  uint32_t d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}

// The MMAs of one K-chunk (KS k-steps) for this warpgroup's m64 block: one m64 x NT MMA per product, A_p x B_q accumulating into
// order group g = p + q (NT / 2 registers each: g0 = hi*hi, g1 = hi*mid + mid*hi, g2 = hi*lo + mid*mid + lo*hi).  Keeping each
// order in its own accumulator keeps the accumulator's rounding 2^-8g smaller on the correction terms, and the epilogue adds the
// groups small-to-large in fp32.  Every MMA writes exactly one group's registers: ptxas only keeps wgmmas in flight back to back
// when their accumulator ranges are identical or disjoint (partly overlapping ranges get a wait after every instruction).
// Tile width, product count, operand major-ness and k-step count are template parameters: a run-time choice between wgmma
// sequences, or a run-time trip count, puts the instructions on paths where the compiler serialises them.
template <int NT, int NPROD, int TRANS, int KS, int NACC>
__device__ __forceinline__ void mma_chunk(float (&acc)[NACC], uint32_t sbase, uint32_t a_off, uint32_t b_off, uint32_t a_ks, uint32_t b_ks,
                                          uint32_t a_ks2, uint64_t a_desc, uint64_t b_desc, uint32_t a_ps, uint32_t b_ps, uint32_t m_off) {
  constexpr int NPL = NPROD >= 6 ? 3 : (NPROD >= 3 ? 2 : 1), G = NT / 2;      // planes = order groups; registers per group
  static_assert(NACC == G * NPL, "one accumulator group of NT columns per product order");
#pragma unroll
  for (int k = 0; k < KS; ++k) {
    uint64_t da[NPL], db[NPL];
#pragma unroll
    for (int pl = 0; pl < NPL; ++pl) {
      const uint32_t pa = sbase + (uint32_t)pl * a_ps + a_off + (uint32_t)(k & 1) * a_ks + (uint32_t)(k >> 1) * a_ks2 + m_off;
      const uint32_t pb = sbase + (uint32_t)pl * b_ps + b_off + (uint32_t)k * b_ks;
      da[pl] = desc_at(a_desc, pa);
      db[pl] = desc_at(b_desc, pb);
    }
    // per group, the products in the order of a wide A_p x [B_0 | ..] issue: g1 = A0 B1, A1 B0; g2 = A0 B2, A1 B1, A2 B0
    Wgmma<NT, TRANS>::mma(acc, da[0], db[0]);
    if constexpr (NPL >= 2) Wgmma<NT, TRANS>::mma(acc + G, da[0], db[1]);
    if constexpr (NPL >= 3) Wgmma<NT, TRANS>::mma(acc + 2 * G, da[0], db[2]);
    if constexpr (NPL >= 2) Wgmma<NT, TRANS>::mma(acc + G, da[1], db[0]);
    if constexpr (NPL >= 3) {
      Wgmma<NT, TRANS>::mma(acc + 2 * G, da[1], db[1]);
      Wgmma<NT, TRANS>::mma(acc + 2 * G, da[2], db[0]);
    }
  }
}

// all lanes run it, lane `pred` arrives: a predicated instruction, not a branch (a divergent block between the wgmmas of a chunk
// makes the compiler wait for every wgmma)
__device__ __forceinline__ void mbar_arrive_if(uint32_t bar, bool pred) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.u32 p, %1, 0;\n\t"
      "@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t"
      "}" ::"r"(bar), "r"((uint32_t)pred)
      : "memory");
}
// trace stamp with the same rule: every lane reads the clock, lane `pred` stores
__device__ __forceinline__ void stamp_if(long long* dst, bool pred) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      ".reg .u64 t;\n\t"
      "mov.u64 t, %%clock64;\n\t"
      "setp.ne.u32 p, %1, 0;\n\t"
      "@p st.global.u64 [%0], t;\n\t"
      "}" ::"l"(dst), "r"((uint32_t)pred)
      : "memory");
}

// MMA side of one tile with tile width NT, NPROD products and KS k-steps per K-chunk and TRANS = MN-major operands: mainloop
// over the tile's K-chunks, then the sums either into the handoff buffer `acc_buf` (handoff: nb = tiles handed off so far) or,
// in place, to one row per lane.  `s` / `ph`: ring slot and per-slot phase bits, carried by the caller across tiles.  body(g, x)
// runs the in-place epilogue of column group g of this thread's row (x = its 32 accumulator sums).
// ctrace: this warp's chunk stamps (nullptr: none), gc: the CTA's chunk counter, the index the producer stamps use.
template <int NT, int NPROD, int TRANS, int KS, class Body>
__device__ __forceinline__ void consume_tile(const CgProblem& P, const Tile& ti, uint32_t ring, uint32_t stg, int slot_bytes, int nstages, uint32_t& s,
                                             uint32_t& ph, uint64_t* bar_full, uint64_t* bar_empty, bool nomma, long long* ctrace, uint32_t& gc,
                                             bool handoff, uint32_t acc_buf, uint32_t& nb, uint64_t* acc_full, uint64_t* acc_empty, Body&& body) {
  constexpr int NGRP = NPROD >= 6 ? 3 : (NPROD >= 3 ? 2 : 1);     // accumulator column groups (product orders)
  constexpr int NACC = NT / 2 * NGRP;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wg = warp >> 2, wl = warp & 3, half = wl >> 1;
  float acc[NACC];
#pragma unroll
  for (int j = 0; j < NACC; ++j) acc[j] = 0.f;
  const uint32_t a_ps = (uint32_t)P.a_pstride, b_ps = (uint32_t)P.b_pstride, a_off = P.a_off, b_off = P.b_off, a_ks = P.a_kstep, b_ks = P.b_kstep;
  const uint32_t a_ks2 = P.a_kstep2;
  const uint64_t a_desc = P.a_desc, b_desc = P.b_desc;
  const uint32_t m_off = (uint32_t)wg * (uint32_t)P.a_moff;     // rows [64 wg, 64 wg + 64) of the A tile
  // One chunk's MMAs stay in flight while the next chunk is awaited and issued; the slot of chunk c - 1 is released once
  // wait_group 1 in chunk c has seen them finish.  Every lane runs the same instructions from the fence to the release: the
  // release and the stamps are predicated, not branched on (see mbar_arrive_if).
  // B2G_CG_DEBUG=2 (no MMA) takes a loop of its own: a branch inside the chunk loop would serialise the wgmmas as well.
  uint32_t prev = 0;
  if (nomma) {
    for (int c = ti.c_begin; c < ti.c_end; ++c, ++gc) {
      mbar_wait(smem_u32(&bar_full[s]), (ph >> s) & 1u);
      mbar_arrive_if(smem_u32(&bar_empty[s]), lane == 0);
      ph ^= 1u << s;
      if (++s == (uint32_t)nstages) s = 0;
    }
  } else {
    for (int c = ti.c_begin; c < ti.c_end; ++c, ++gc) {
      long long* const tr = ctrace + gc * 8;
      const bool stamp = ctrace != nullptr && lane == 0 && gc < 64;
      stamp_if(tr + 3, stamp);
      mbar_wait(smem_u32(&bar_full[s]), (ph >> s) & 1u);
      stamp_if(tr + 4, stamp);
      wg_arrive();
      mma_chunk<NT, NPROD, TRANS, KS>(acc, ring + s * (uint32_t)slot_bytes, a_off, b_off, a_ks, b_ks, a_ks2, a_desc, b_desc, a_ps, b_ps, m_off);
      wg_commit();
      wg_wait<1>();
      mbar_arrive_if(smem_u32(&bar_empty[prev]), lane == 0 && c > ti.c_begin);      // chunk c - 1's slot may be refilled
      stamp_if(tr + 5, stamp);
      prev = s;
      ph ^= 1u << s;
      if (++s == (uint32_t)nstages) s = 0;
    }
    wg_wait<0>();
    mbar_arrive_if(smem_u32(&bar_empty[prev]), lane == 0);
  }
  // correction column groups, smallest order first
  if constexpr (NGRP > 2) {
#pragma unroll
    for (int j = 0; j < NT / 2; ++j) acc[j] = acc[j] + (acc[j + NT / 2] + acc[j + NT]);
  } else if constexpr (NGRP > 1) {
#pragma unroll
    for (int j = 0; j < NT / 2; ++j) acc[j] = acc[j] + acc[j + NT / 2];
  }
  if (handoff) {
    // Buffer rows of NT fp32, the 16-byte chunks of row R XOR-swizzled by R & 7: the fragment stores (8 rows x 2 chunks per
    // instruction) and the epilogue's row reads (8 rows per 128-byte phase) both spread over all banks.  The buffer is free once
    // the epilogue warpgroup has read the previous handed-off tile.
    mbar_wait(smem_u32(acc_empty), (nb & 1u) ^ 1u);
    const uint32_t R = 64u * wg + 16u * wl + (uint32_t)(lane >> 2), sw = (uint32_t)(lane >> 2);      // sw = R & 7 (= (R + 8) & 7)
    const uint32_t rowa = acc_buf + R * (uint32_t)(NT * 4) + (uint32_t)((lane & 1) * 8);
#pragma unroll
    for (int j = 0; j < NT / 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t a = rowa + (uint32_t)h * (8u * NT * 4) + ((((uint32_t)(2 * j) + (uint32_t)((lane & 3) >> 1)) ^ sw) << 4);
        asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(a), "f"(acc[4 * j + 2 * h]), "f"(acc[4 * j + 2 * h + 1]) : "memory");
      }
    __syncwarp();
    mbar_arrive_if(smem_u32(acc_full), lane == 0);
    ++nb;
    return;
  }
  // In place: fragments -> one row per lane, 16 columns at a time through the warpgroup's staging block (rows of 64 B, 16-byte chunks
  // XOR-swizzled by row pair).  Warp wl & 1 of a warpgroup owns rows 32 (wl & 1) .. + 31 and `half` the parity of its column
  // groups; a pair of column groups (64 columns) is gathered in four steps, then every warp runs the epilogue of its group.
  const int rrow = 32 * (wl & 1) + lane;
  const uint32_t wstg = stg + (uint32_t)wg * 4096u;
#pragma unroll
  for (int R = 0; R < (NT + 63) / 64; ++R) {
    float x[32];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int c0 = 64 * R + 16 * t;              // first column of this step: group 2R + (t >> 1), columns 16 (t & 1) .. of it
      if (c0 < NT) {
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");     // the previous step's readers are done
#pragma unroll
        for (int jj = 0; jj < 2; ++jj)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = 16 * wl + (lane >> 2) + 8 * h, chunk = 2 * jj + ((lane & 3) >> 1);
            const int j = c0 / 8 + jj;
            const uint32_t a = wstg + (uint32_t)row * 64u + (uint32_t)((chunk ^ ((row >> 1) & 3)) << 4) + (uint32_t)((lane & 1) * 8);
            asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(a), "f"(acc[4 * j + 2 * h]), "f"(acc[4 * j + 2 * h + 1]) : "memory");
          }
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
        if (half == (t >> 1)) {
#pragma unroll
          for (int cc = 0; cc < 4; ++cc) {
            const uint32_t a = wstg + (uint32_t)rrow * 64u + (uint32_t)((cc ^ ((rrow >> 1) & 3)) << 4);
            float* xd = x + 16 * (t & 1) + 4 * cc;
            asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(xd[0]), "=f"(xd[1]), "=f"(xd[2]), "=f"(xd[3]) : "r"(a));
          }
        }
      }
    }
    const int g = 2 * R + half;
    if (32 * g < NT) body(g, x);
  }
}

// per-problem constants of one output row r of a tile: the row's offsets inside a tile (the r -> (i0, i1, i2) decomposition needs
// integer divisions), recomputed only when a role moves to another problem
struct RowOff {
  long long roff = 0, rmoff = 0;
  int ri0 = 0, ri1 = 0;
  bool ok = true;                                    // not cut by lim_i0
  __device__ __forceinline__ void set(const CgProblem& Q, int r) {
    const int d0 = Q.d0, d1 = Q.d1;
    const int i0 = r % d0, i12 = r / d0, i1 = i12 % d1, i2 = i12 / d1;
    roff = Q.o_base + (long long)i0 * Q.o0 + (long long)i1 * Q.o1 + (long long)i2 * Q.o2;
    if (Q.rgrp_rows > 0) roff += Q.rgrp_off[min(r / Q.rgrp_rows, 7)];
    rmoff = Q.m_base + (long long)i0 * Q.m0 + (long long)i1 * Q.m1 + (long long)i2 * Q.m2;
    ri0 = i0; ri1 = i1;
    ok = Q.lim_i0 <= 0 || i0 < Q.lim_i0;
  }
};

// 16 warps per CTA: 128 registers per thread at launch, then MMA_REGS / EPI_REGS / PROD_REGS.
__global__ void __launch_bounds__(NTHREADS, 1)
cg_kernel(const __grid_constant__ CgPack pk, int nprob, int total_tiles, const CUtensorMap* __restrict__ maps, int max_stages,
          int dbg, long long* __restrict__ trace) {
  const CgProblem* __restrict__ probs = pk.p;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_full[CG_MAX_STAGES], bar_empty[CG_MAX_STAGES], acc_full, acc_empty;
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);          // warp-uniform for the compiler, not just in fact
  const int trace_cta = dbg >> 8;                    // bring-up: the CTA whose roles write clock stamps
  const bool dbg_noload = dbg & 1, dbg_nomma = dbg & 2, dbg_nostore = dbg & 4, dbg_nost = dbg & 16;    // 16: epilogue math without the global stores
  if (tid == 0) {
    for (int s = 0; s < max_stages; ++s) { mbar_init(smem_u32(&bar_full[s]), 1); mbar_init(smem_u32(&bar_empty[s]), NMMA_WARPS); }
    mbar_init(smem_u32(&acc_full), NMMA_WARPS);
    mbar_init(smem_u32(&acc_empty), NEPI_WARPS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const uint32_t stg = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t ring = stg + STG_BYTES;
  pdl_trigger();
  pdl_wait();

  if (warp >= PROD_WARP0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PROD_REGS));
    const int pw = warp - PROD_WARP0;
    if (pw >= NPROD_WARPS) return;
    // ============================================================================================ TMA producers
    {
      // Ring slot s and the phase parity of every slot (bit s of ph): the partition of the ring (slot size, slot count) belongs
      // to the problem, so a slot's barrier may have completed a different number of phases than its neighbours'.
      uint32_t gc = 0, s = 0, ph = 0, nbuf = 0;        // nbuf: handed-off tiles so far
      int slot_bytes = 0, nstages = 1;
      bool handoff = false;
      Walker w;
      int n2 = 1, nloads = 0, planes = 0, tx = 0;
      const int* tab = nullptr;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        if (w.advance(probs, nprob, tile)) {
          const CgProblem& P = probs[w.p];
          n2 = P.n2; nloads = P.nloads; planes = P.planes; tx = P.tx_bytes; tab = P.tm_tab; handoff = cg_epi_handoff(P.epi);
          if (P.slot_bytes != slot_bytes || P.nstages != nstages) {
            // new partition: every slot of the old one must have been consumed before its bytes are overwritten (a fresh
            // barrier passes the parity-1 wait at once, so never-used slots cost nothing), and the new ring may cover the
            // old handoff buffer: wait until the MMA warps have handed off the last tile (acc_full has completed nbuf phases;
            // with the ring drained it is at most one behind) and the epilogue warpgroup has read it (acc_empty likewise)
            for (int q = 0; q < nstages; ++q) mbar_wait(smem_u32(&bar_empty[q]), ((ph >> q) & 1u) ^ 1u);
            if (nbuf) {
              mbar_wait(smem_u32(&acc_full), (nbuf - 1) & 1u);
              mbar_wait(smem_u32(&acc_empty), (nbuf - 1) & 1u);
              asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // its generic reads before our TMA writes
            }
            slot_bytes = P.slot_bytes; nstages = P.nstages; s = 0;
          }
        }
        const Tile ti = w.tile(tile);
        const CgProblem& P = probs[ti.p];
        if (handoff && ti.c_end > ti.c_begin) ++nbuf;
        if (P.dep_ctr) {                                                 // fused layers: wait for the tiles this one reads
          const int* __restrict__ ctr = P.dep_ctr;
          const int x0 = P.dep_by_chunk ? ti.c_begin : ti.tm, x1 = P.dep_by_chunk ? ti.c_end : ti.tm + 1;
          const int lo = x0 * P.dep_rows / P.dep_rows_tile, hi = min(P.dep_tiles - 1, (x1 * P.dep_rows - 1) / P.dep_rows_tile);
          const int expect = P.dep_expect * NEPI_WARPS;
          for (int j = lo + lane; j <= hi; j += 32) {
            int seen;
            do {
              asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(seen) : "l"(ctr + j) : "memory");
              if (seen < expect) __nanosleep(100);
            } while (seen < expect);
          }
          __syncwarp();
          asm volatile("fence.proxy.async.global;" ::: "memory");
        }
        // per-tile box origins: everything but the chunk terms
        int base[CG_MAX_LOADS][5];
#pragma unroll
        for (int l = 0; l < CG_MAX_LOADS; ++l) {
          if (l < nloads) {
            const CgLoad& L = P.ld[l];
#pragma unroll
            for (int d = 0; d < 5; ++d) base[l][d] = L.c0[d] + ti.tm * L.d_tm[d] + ti.tn * L.d_tn[d];
            if (tab) { base[l][1] += tab[(ti.tm * CG_MAX_LOADS + l) * 2]; base[l][2] += tab[(ti.tm * CG_MAX_LOADS + l) * 2 + 1]; }
          }
        }
        int c1 = n2 > 1 ? ti.c_begin / n2 : 0, c2 = ti.c_begin - c1 * n2;
        for (int c = ti.c_begin; c < ti.c_end; ++c, ++gc) {
          const bool tr = trace && blockIdx.x == trace_cta && pw == 0 && gc < 64 && lane == 0;
          if (tr) trace[gc * 8 + 0] = clock64();
          mbar_wait(smem_u32(&bar_empty[s]), ((ph >> s) & 1u) ^ 1u);
          if (tr) trace[gc * 8 + 1] = clock64();
          const uint32_t full = smem_u32(&bar_full[s]);
          const bool leader = elect_one();
          if (dbg_noload) { if (pw == 0 && leader) mbar_arrive(full); }
          else {
            if (pw == 0 && leader) mbar_expect_tx(full, (uint32_t)tx);        // the one arrival of the phase; boxes may land before it
            const uint32_t sbase = ring + s * (uint32_t)slot_bytes;
            int j = 0;                                                 // box index inside the chunk, dealt round-robin to the producer warps
#pragma unroll
            for (int l = 0; l < CG_MAX_LOADS; ++l) {
              if (l < nloads) {
                const CgLoad& L = P.ld[l];
                int crd[5];
#pragma unroll
                for (int d = 0; d < 5; ++d) crd[d] = base[l][d] + c1 * L.d_c1[d] + c2 * L.d_c2[d];
                if (L.plane_box) {                               // all planes in one box (plane = outermost coordinate, 0)
                  if ((j & (NPROD_WARPS - 1)) == pw && leader) tma_load(sbase + (uint32_t)L.smem_off, maps + L.map, full, L.rank, crd);
                  ++j;
                } else {
                  for (int pl = 0; pl < planes; ++pl, ++j) {
#pragma unroll
                    for (int d = 2; d < 5; ++d) if (d == L.rank - 1) crd[d] = pl;
                    if ((j & (NPROD_WARPS - 1)) == pw && leader)
                      tma_load(sbase + (uint32_t)(pl * L.plane_stride + L.smem_off), maps + L.map, full, L.rank, crd);
                  }
                }
              }
            }
          }
          if (tr) { trace[gc * 8 + 2] = clock64(); trace[gc * 8 + 6] = ti.p * 100000 + ti.tm * 10 + ti.tn; }
          if (++c2 == n2) { c2 = 0; ++c1; }
          ph ^= 1u << s;
          if (++s == (uint32_t)nstages) s = 0;
        }
      }
    }
  } else if (warp < NMMA_WARPS) {
    // ============================================================================================ MMA warpgroups
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(MMA_REGS));
    const int q = 2 * (warp >> 2) + (warp & 1);
    uint32_t it = 0, s = 0, ph = 0, gc = 0, nb = 0;      // nb: tiles handed off to the epilogue warpgroup so far
    int slot_bytes = 0, nstages = 1;
    Walker w;
    long long* const ctrace = trace && blockIdx.x == trace_cta && warp == 0 ? trace : nullptr;     // chunk stamps: first MMA warp
    const int r = q * 32 + lane;                         // output row of this thread in the in-place epilogue
    int epi = 0, rows_tile = 0, lim_rows = 0, umma_n = 0, n_valid = 0, shape = 0;
    bool handoff = false;
    uint32_t acc_buf = 0;
    long long o_tm = 0;
    RowOff ro;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      if (w.advance(probs, nprob, tile)) {
        const CgProblem& Q = probs[w.p];
        epi = Q.epi; rows_tile = Q.rows_tile; lim_rows = Q.lim_rows; umma_n = Q.umma_n; n_valid = Q.n_valid; o_tm = Q.o_tm;
        ro.set(Q, r);
        shape = cg_shape_key(Q.umma_n, Q.nprod, Q.mn_major != 0, Q.ksteps);
        if (Q.slot_bytes != slot_bytes || Q.nstages != nstages) { slot_bytes = Q.slot_bytes; nstages = Q.nstages; s = 0; }
        handoff = cg_epi_handoff(epi);
        acc_buf = ring + (uint32_t)(nstages * slot_bytes);
      }
      const Tile ti = w.tile(tile);
      if (ti.c_end <= ti.c_begin) continue;
      const CgProblem& P = probs[ti.p];
      const bool valid0 = r < rows_tile && ti.tm * rows_tile + r < lim_rows && ro.ok;
      const long long off0 = ro.roff + (long long)ti.tm * o_tm;
      const int n0 = ti.tn * umma_n;
      const bool tre = trace && blockIdx.x == trace_cta && warp == 0 && lane == 0 && it < 16;
      if (tre) trace[512 + it * 4 + 0] = clock64();
      // in-place epilogue (RAW / WGRAD) of column group g of this thread's row.  Every lane owns one output row and writes its
      // 32 columns itself (128 B of fp32): 16-byte vector stores or red.adds.
      auto body = [&](int g, float (&x)[32]) {
        const int ng = n0 + 32 * g;                      // first problem column of the group
        if (dbg_nostore || ng >= n_valid || !valid0) return;
        float* dst = P.out_f + off0 + (long long)(ng >> 5) * P.f_grp;
        if (epi == CG_EPI_RAW) {
          if (P.atomic) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
              asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(dst + 4 * j), "f"(x[4 * j]), "f"(x[4 * j + 1]), "f"(x[4 * j + 2]),
                           "f"(x[4 * j + 3])
                           : "memory");
          } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) *reinterpret_cast<float4*>(dst + 4 * j) = make_float4(x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]);
          }
          return;
        }
        // CG_EPI_WGRAD
        const float sc = P.scale;
        if (P.atomic) {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(dst + 4 * j), "f"(x[4 * j] * sc), "f"(x[4 * j + 1] * sc),
                         "f"(x[4 * j + 2] * sc), "f"(x[4 * j + 3] * sc)
                         : "memory");
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<float4*>(dst + 4 * j) = make_float4(x[4 * j] * sc, x[4 * j + 1] * sc, x[4 * j + 2] * sc, x[4 * j + 3] * sc);
          if (P.dp_n > 1) {                          // final values: push them to their owner now (posted NVLink stores)
            const int i4 = (int)((dst - P.dp_gbase) >> 2), per4 = P.dp_per4;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int owner = (i4 + j) / per4;
              if (owner != P.dp_rank)
                reinterpret_cast<float4*>(P.dp_recv[owner])[(size_t)P.dp_rank * per4 + (i4 + j - owner * per4)] =
                    make_float4(x[4 * j] * sc, x[4 * j + 1] * sc, x[4 * j + 2] * sc, x[4 * j + 3] * sc);
            }
          }
        }
      };
#define CG_CONSUME(NT, NPROD, TRANS, KS)                                                                                                      \
  consume_tile<NT, NPROD, TRANS, KS>(P, ti, ring, stg, slot_bytes, nstages, s, ph, bar_full, bar_empty, dbg_nomma, ctrace, gc, handoff, acc_buf, \
                                     nb, &acc_full, &acc_empty, body)
      // the (width, products, major-ness, k-steps) combinations cg_shape_supported() admits on the host; anything else is a bug: trap
      switch (shape) {
        case cg_shape_key(32, 6, false, 4): CG_CONSUME(32, 6, 0, 4); break;
        case cg_shape_key(64, 6, false, 4): CG_CONSUME(64, 6, 0, 4); break;
        case cg_shape_key(64, 3, false, 4): CG_CONSUME(64, 3, 0, 4); break;
        case cg_shape_key(128, 3, false, 4): CG_CONSUME(128, 3, 0, 4); break;
        case cg_shape_key(64, 3, true, 4): CG_CONSUME(64, 3, 1, 4); break;
        case cg_shape_key(64, 3, true, 9): CG_CONSUME(64, 3, 1, 9); break;
        case cg_shape_key(128, 3, true, 4): CG_CONSUME(128, 3, 1, 4); break;
        default: __trap();
      }
#undef CG_CONSUME
      if (tre) {
        trace[512 + it * 4 + 1] = clock64();
        trace[512 + it * 4 + 2] = handoff;
        trace[512 + it * 4 + 3] = ti.p * 100000 + ti.tm * 10 + ti.tn;
      }
      ++it;
    }
  } else {
    // ============================================================================================ epilogue warpgroup
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(EPI_REGS));
    const int ew = warp - EPI_WARP0;
    const int r = ew * 32 + lane;                        // output row of this thread
    uint32_t ne = 0;                                     // handed-off tiles finished so far
    int slot_bytes = 0, nstages = 1;
    Walker w;
    // per-problem constants of this thread, recomputed only when the CTA moves to another problem
    int epi = 0, rows_tile = 0, lim_rows = 0, umma_n = 0, out_planes = 0, grp_stride = 32, n_valid = 0, grp_tab = 0;
    bool handoff = false;
    uint32_t acc_buf = 0;
    long long o_tm = 0, m_tm = 0;
    RowOff ro;
    const float* __restrict__ bias = nullptr;
    const uint16_t* __restrict__ mask = nullptr;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      if (w.advance(probs, nprob, tile)) {
        const CgProblem& Q = probs[w.p];
        epi = Q.epi; rows_tile = Q.rows_tile; lim_rows = Q.lim_rows; umma_n = Q.umma_n; out_planes = Q.out_planes;
        grp_stride = Q.grp_stride; n_valid = Q.n_valid; o_tm = Q.o_tm; m_tm = Q.m_tm; bias = Q.bias; mask = Q.mask; grp_tab = Q.grp_tab;
        ro.set(Q, r);
        if (Q.slot_bytes != slot_bytes || Q.nstages != nstages) { slot_bytes = Q.slot_bytes; nstages = Q.nstages; }
        handoff = cg_epi_handoff(epi);
        acc_buf = ring + (uint32_t)(nstages * slot_bytes);
      }
      const Tile ti = w.tile(tile);
      if (ti.c_end <= ti.c_begin || !handoff) continue;
      const CgProblem& P = probs[ti.p];
      bool valid0 = r < rows_tile && ti.tm * rows_tile + r < lim_rows && ro.ok;
      long long off0 = ro.roff + (long long)ti.tm * o_tm;
      const long long moff0 = ro.rmoff + (long long)ti.tm * m_tm;
      if (P.tm_sub > 1) {                              // band tr of block tq (cg.cuh: tm_sub)
        const int tq = ti.tm / P.tm_sub, tr = ti.tm - tq * P.tm_sub;
        off0 = ro.roff + (long long)tq * o_tm + (long long)tr * P.o_sub;
        valid0 = valid0 && tr * P.d1 + ro.ri1 < P.lim_i1;
      }
      const int n0 = ti.tn * umma_n, ngroups = umma_n >> 5;
      // the row limits and output / mask offsets of column group g (per group from the tables for grp_tab problems)
      auto group_at = [&](int g, bool& valid, long long& off, long long& moff) {
        const int ng = n0 + 32 * g;
        valid = valid0; off = off0; moff = moff0;
        if (grp_tab) {
          const int gg = ng >> 5;
          valid = valid0 && ro.ri0 < P.grp_lim0[gg] && ro.ri1 < P.grp_lim1[gg];
          off = off0 + P.grp_off[gg]; moff = moff0 + P.grp_moff[gg] - ng;     // (the mask load adds ng)
        }
      };
      const bool tre = trace && blockIdx.x == trace_cta && ew == 0 && lane == 0 && ne < 16;
      if (tre) trace[576 + ne * 4 + 0] = clock64();
      // DGRAD: the ReLU mask does not depend on the sums, so its loads are issued before the handoff wait, while the MMA
      // warps are still in the mainloop; bit c of mbits[g] = column 32g + c of this row is kept (an invalid row keeps none).
      // Four groups: the instantiated tile widths are at most 128.
      uint32_t mbits[4] = {0u, 0u, 0u, 0u};
      if (epi == CG_EPI_DGRAD && !dbg_nostore) {
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          bool valid;
          long long off, moff;
          group_at(g, valid, off, moff);
          const int ng = n0 + 32 * g;
          if (g < ngroups && valid && ng < n_valid) {
            uint4 mk[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) mk[j] = __ldg(reinterpret_cast<const uint4*>(mask + moff + ng) + j);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const uint32_t wd[4] = {mk[j].x, mk[j].y, mk[j].z, mk[j].w};
#pragma unroll
              for (int uu = 0; uu < 4; ++uu) {
                if (wd[uu] & 0x00007FFFu) mbits[g] |= 1u << (8 * j + 2 * uu);
                if (wd[uu] & 0x7FFF0000u) mbits[g] |= 1u << (8 * j + 2 * uu + 1);
              }
            }
          }
        }
      }
      mbar_wait(smem_u32(&acc_full), ne & 1u);
      if (tre) trace[576 + ne * 4 + 1] = clock64();
      const bool split_fin = P.ws != nullptr;          // split-K tile of an ACT problem: partial sums first, the last arriver finishes
      float* __restrict__ wsrow = split_fin ? P.ws + ((size_t)(ti.tm * w.tiles_n + ti.tn) * 128 + r) * umma_n : nullptr;
      // epilogue of column group g of this thread's row; pass 0: x = this tile's accumulator sums, pass 1: x = the finished
      // split-K sums read back by the last arriver
      auto body = [&](int g, float (&x)[32], int pass) {
        const int ng = n0 + 32 * g;                      // first problem column of the group
        bool valid;
        long long off, moff;
        group_at(g, valid, off, moff);
        if (pass == 0 && split_fin) {                    // partial sums of this split -> workspace
#pragma unroll
          for (int j = 0; j < 8; ++j)
            asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(wsrow + 32 * g + 4 * j), "f"(x[4 * j]), "f"(x[4 * j + 1]), "f"(x[4 * j + 2]),
                         "f"(x[4 * j + 3])
                         : "memory");
          return;
        }
        const bool live = !dbg_nostore && ng < n_valid;
        float4 bv[8];
        if (epi == CG_EPI_ACT && live) {
#pragma unroll
          for (int j = 0; j < 8; ++j) bv[j] = __ldg(reinterpret_cast<const float4*>(bias + (long long)(ng >> 5) * P.bias_grp) + j);
        }
        if (!live) return;
        if (epi == CG_EPI_ACT) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            x[4 * j] = fmaxf(x[4 * j] + bv[j].x, 0.f); x[4 * j + 1] = fmaxf(x[4 * j + 1] + bv[j].y, 0.f);
            x[4 * j + 2] = fmaxf(x[4 * j + 2] + bv[j].z, 0.f); x[4 * j + 3] = fmaxf(x[4 * j + 3] + bv[j].w, 0.f);
          }
          if (P.f0 > 0 && valid && !dbg_nost) {        // optional fp32 copy (cnn_fc1 features for the head kernels)
            float* dst = P.out_f + (long long)ti.tm * P.f_tm + (long long)r * P.f0 + (long long)(ng >> 5) * P.f_grp;
#pragma unroll
            for (int j = 0; j < 8; ++j) *reinterpret_cast<float4*>(dst + 4 * j) = make_float4(x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]);
          }
        } else {   // CG_EPI_DGRAD: ReLU mask = hi plane of the forward activation at the same position
          const uint32_t mb = g == 0 ? mbits[0] : g == 1 ? mbits[1] : g == 2 ? mbits[2] : mbits[3];
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (!((mb >> j) & 1u)) x[j] = 0.f;
          if (P.colsum) {
            // bias gradient: column sums over this warp's 32 rows (invalid rows are zero: their mask words were not loaded) by a
            // transposing butterfly -- 31 shuffles leave lane c with the sum of column c -- then one 128-byte red.add per warp
            float cs[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) cs[j] = x[j];
#pragma unroll
            for (int wd = 16; wd >= 1; wd >>= 1) {
              const bool up = (lane & wd) != 0;
#pragma unroll
              for (int j = 0; j < wd; ++j) {
                const float send = up ? cs[j] : cs[j + wd], keep = up ? cs[j + wd] : cs[j];
                cs[j] = keep + __shfl_xor_sync(0xffffffffu, send, wd);
              }
            }
            atomicAdd(P.colsum + ((ng + lane) & P.colsum_mask), cs[0]);
          }
        }
        // ---- BF16 planes: hi = bf16(x), then the residual feeds the next plane
        const long long gcol = grp_tab ? 0 : (long long)(ng >> 5) * grp_stride;
        const long long roff = off + gcol;
        const int q0 = lane & ~3, qi = lane & 3;           // this lane's quad, and its place in it
#pragma unroll 1
        for (int pl = 0; pl < out_planes; ++pl) {
          uint32_t pk[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            pk[j] = pack_bf16x2(x[2 * j], x[2 * j + 1]);
            x[2 * j] -= __uint_as_float(pk[j] << 16);
            x[2 * j + 1] -= __uint_as_float(pk[j] & 0xFFFF0000u);
          }
          if (dbg_nost) continue;
          // The row's 64 bytes are 4 16-byte chunks, pk[4c .. 4c + 3] = chunk c.  A 4 x 4 transpose of the chunks inside each quad
          // of lanes (two shfl_xor exchange steps) leaves lane q0 + i holding chunk i of rows q0 .. q0 + 3 in slots 0 .. 3, so that
          // store j writes 8 rows (q0 + j of every quad) with 64 contiguous bytes each: 8 whole row segments per instruction instead
          // of 32 rows' quarter segments (half 32-byte sectors).
#pragma unroll
          for (int m = 1; m <= 2; m <<= 1) {
            const bool up = (lane & m) != 0;
#pragma unroll
            for (int c0 = 0; c0 < 4; ++c0) {
              if (c0 & m) continue;
              const int c1 = c0 | m;                   // slot c of lane i moves to lane i ^ m, slot c ^ m, where bit m of i and c differ
#pragma unroll
              for (int u = 0; u < 4; ++u) {
                const uint32_t got = __shfl_xor_sync(0xffffffffu, up ? pk[4 * c0 + u] : pk[4 * c1 + u], m);
                if (up) pk[4 * c0 + u] = got; else pk[4 * c1 + u] = got;
              }
            }
          }
          uint16_t* const base = P.out_p[pl];
#pragma unroll
          for (int j = 0; j < 4; ++j) {                  // row q0 + j: its owner's offset and limit
            const long long oj = __shfl_sync(0xffffffffu, roff, q0 + j);
            const bool vj = __shfl_sync(0xffffffffu, valid ? 1 : 0, q0 + j) != 0;
            if (vj) *reinterpret_cast<uint4*>(base + oj + 8 * qi) = make_uint4(pk[4 * j], pk[4 * j + 1], pk[4 * j + 2], pk[4 * j + 3]);
          }
        }
      };
      // this thread's row of the handoff buffer (16-byte chunk c of row r at c ^ (r & 7), see consume_tile), one 32-column group
      // at a time; the buffer is released as soon as the last group is in registers
      const uint32_t rowa = acc_buf + (uint32_t)(r * umma_n * 4), sw = (uint32_t)(r & 7);
      for (int g = 0; g < ngroups; ++g) {
        float x[32];
#pragma unroll
        for (int cc = 0; cc < 8; ++cc) {
          const uint32_t a = rowa + ((((uint32_t)(8 * g + cc)) ^ sw) << 4);
          asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(x[4 * cc]), "=f"(x[4 * cc + 1]), "=f"(x[4 * cc + 2]), "=f"(x[4 * cc + 3]) : "r"(a));
        }
        if (g == ngroups - 1) {
          __syncwarp();
          mbar_arrive_if(smem_u32(&acc_empty), lane == 0);
        }
        body(g, x, 0);
      }
      ++ne;
      bool last_arriver = !split_fin;
      if (split_fin) {
        __syncwarp();
        int old = 0;
        if (lane == 0) { __threadfence(); old = atomicAdd(P.ws_cnt + (ti.tm * w.tiles_n + ti.tn) * NEPI_WARPS + ew, 1); }
        old = __shfl_sync(0xffffffffu, old, 0);
        last_arriver = old == w.splits - 1;
        if (last_arriver) {                              // the complete sums, and a clean workspace for the next step
          __threadfence();
          if (lane == 0) P.ws_cnt[(ti.tm * w.tiles_n + ti.tn) * NEPI_WARPS + ew] = 0;     // next step starts from zero
          for (int g = 0; g < ngroups; ++g) {
            float x[32];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float4 sum = __ldcg(reinterpret_cast<const float4*>(wsrow + 32 * g) + j);
              x[4 * j] = sum.x; x[4 * j + 1] = sum.y; x[4 * j + 2] = sum.z; x[4 * j + 3] = sum.w;
              __stcg(reinterpret_cast<float4*>(wsrow + 32 * g) + j, make_float4(0.f, 0.f, 0.f, 0.f));
            }
            body(g, x, 1);
          }
        }
      }
      __syncwarp();
      if (lane == 0 && P.done_ctr && last_arriver) {     // this warp's rows of the tile are in global memory
        __threadfence();
        atomicAdd(P.done_ctr + ti.tm, 1);
      }
      if (tre) { trace[576 + (ne - 1) * 4 + 2] = clock64(); trace[576 + (ne - 1) * 4 + 3] = ti.p * 100000 + ti.tm * 10 + ti.tn; }
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

}  // namespace

// ring budget (cg_finalize): the dynamic part minus the in-place epilogue staging; the kernel's static shared memory (barriers) takes < 1 KiB
// of the 227 KiB
bool cg_shape_supported(int umma_n, int nprod, bool mn_major, int ksteps) {
  switch (cg_shape_key(umma_n, nprod, mn_major, ksteps)) {
    case cg_shape_key(32, 6, false, 4): case cg_shape_key(64, 6, false, 4): case cg_shape_key(64, 3, false, 4): case cg_shape_key(128, 3, false, 4):
    case cg_shape_key(64, 3, true, 4): case cg_shape_key(64, 3, true, 9): case cg_shape_key(128, 3, true, 4): return true;
    default: return false;
  }
}

int cg_smem_limit() { return 226 * 1024 - STG_BYTES; }

int cg_encode_map(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                  const uint32_t* elem_strides, int swizzle) {
  if (swizzle != 128 && swizzle != 64) return -1;
  if (!g_encode) {
    cudaDriverEntryPointQueryResult q;
    void* fn = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn || q != cudaDriverEntryPointSuccess) return -1;
    g_encode = (EncodeTiledFn)fn;
  }
  cuuint64_t gd[5], gs[5];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = elem_strides ? elem_strides[i] : 1; }
  for (int i = 0; i + 1 < rank; ++i) gs[i] = strides_bytes[i];
  const CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              swizzle == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

// wgmma descriptor (wgmma.cuh): LBO >> 4 in [16,30), SBO >> 4 in [32,46), swizzle mode in [62,64) (1 = 128 B, 2 = 64 B).  Rows of
// `swizzle` bytes in 8-row groups: SBO = 8 rows.  K-major: LBO unused (the k16 slice lies inside one row); MN-major: LBO = stride
// between the swizzle / 2-element atoms along M|N (one TMA box each)
unsigned long long cg_desc_bits(int swizzle, bool mn_major, int lbo) {
  const unsigned long long l = mn_major ? (unsigned)lbo : 16u, sbo = 8u * (unsigned)swizzle;
  return ((l >> 4) & 0x3FFF) << 16 | ((sbo >> 4) & 0x3FFF) << 32 | (unsigned long long)(swizzle == 128 ? 1 : 2) << 62;
}

int cg_finalize(CgGroup& g, int smem_budget) {
  int start = 0, slot = 0;
  g.flops = 0;
  for (int i = 0; i < g.n; ++i) {
    CgProblem& P = g.host[i];
    P.tile_start = start;
    start += P.tiles_m * P.tiles_n * P.splits;
    for (int l = 0; l < P.nloads; ++l) {
      CgLoad& L = P.ld[l];
      L.plane_stride = L.smem_off >= P.b_off ? P.b_pstride : P.a_pstride;
      if (L.plane_box && L.box_bytes != L.plane_stride) return -2;      // stacked planes must land where the MMA descriptors look
    }
    const int need = P.b_off + P.planes * P.b_pstride;
    P.slot_bytes = (need + 1023) / 1024 * 1024;
    slot = slot > P.slot_bytes ? slot : P.slot_bytes;
  }
  g.total_tiles = start;
  const int avail = smem_budget - 1024 /* alignment slack */;
  g.slot_bytes = slot; g.nstages = 0;              // (largest slot; the most stages any problem uses)
  int ring = 0;
  for (int i = 0; i < g.n; ++i) {
    CgProblem& P = g.host[i];
    const int acc = cg_epi_handoff(P.epi) ? cg_acc_bytes(P.umma_n) : 0;     // the handoff buffer follows the problem's ring
    const int avail_ring = avail - acc;
    P.nstages = P.slot_bytes > 0 ? avail_ring / P.slot_bytes : 0;
    if (P.nstages > CG_MAX_STAGES) P.nstages = CG_MAX_STAGES;
    if (P.nstages < 2) return -1;
    P.slot_bytes = avail_ring / P.nstages / 1024 * 1024;   // one slot size per stage count: problems with equal depth share the partition
    g.nstages = g.nstages > P.nstages ? g.nstages : P.nstages;
    ring = ring > P.nstages * P.slot_bytes + acc ? ring : P.nstages * P.slot_bytes + acc;
  }
  g.ring_bytes = ring;
  return 0;
}

long long* g_cg_trace = nullptr;      // bring-up: clock64 stamps of CTA 0 (set by tools through b2g_debug_cg_trace)

cudaError_t cg_launch(const CgGroup& g, const CUtensorMap* dev_maps, int num_sms, cudaStream_t s, bool pdl, int debug_flags) {
  if (g.total_tiles <= 0 || (debug_flags & 8)) return cudaSuccess;     // bit 3: skip the launch (timing ablation)
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(cg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const int smem = 1024 + STG_BYTES + g.ring_bytes;
  const int grid = g.total_tiles < num_sms ? g.total_tiles : num_sms;
  CgPack pk;              // (host staging; the launch copies it into the parameter buffer)
  static_assert(sizeof(CgPack) < 28 * 1024, "problem list must fit the kernel parameter space (32,764 B)");
  for (int i = 0; i < g.n; ++i) pk.p[i] = g.host[i];
  cudaError_t e = launch_pdl(cg_kernel, dim3(grid), dim3(NTHREADS), (size_t)smem, s, pdl, pk, g.n, g.total_tiles, dev_maps, g.nstages, debug_flags, g_cg_trace);
  if (e != cudaSuccess) fprintf(stderr, "cg_launch %s: %s (grid %d, %d threads, smem %d)\n", g.name, cudaGetErrorString(e), grid, NTHREADS, smem);
  return e;
}

}  // namespace b2g
