// TMA-fed wgmma contraction engine ("cg"): declarations shared by cg.cu (kernel) and sac.cu (problem builders).
//
// Every dense contraction of the step is a list of 128-row output tiles; the operands of a tile are fetched, K-chunk by
// K-chunk, by cp.async.bulk.tensor (TMA) boxes over BF16 plane tensors straight into swizzled (128B; 64B for conv1's A at one
// image channel) shared-memory wgmma tiles.  Convolutions need no im2col buffer: their patches / shifted windows / zero borders are expressed as tensor-map
// VIEWS (overlapping strides, element strides, out-of-bound zero fill) of the NHWC activation planes, so two elected
// lanes feed the whole ring (tools/tma_probe.cu checks each view behaviour on the device).  A launch is a list of problems;
// problems of one launch may depend on each other tile by tile (fused layers) and may split K with in-kernel finalisation.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2g {

constexpr int CG_MAX_LOADS = 4;     // TMA boxes per K-chunk and plane (A atoms + B atoms)
constexpr int CG_MAX_PROBLEMS = 16; // problems per grouped launch (the whole list travels as a __grid_constant__ kernel parameter)
constexpr int CG_MAX_STAGES = 8;
constexpr int CG_MAX_PLANES = 3;
constexpr int CG_EPI_WARPS = 4;    // the epilogue warpgroup's warps (one output row per lane); each signals a finished tile once
                                   // (dependency counters, split-K arrival counters)

enum CgEpiKind : int {
  CG_EPI_ACT = 0,     // relu(acc + bias[n]) -> BF16 planes (activations; optional fp32 copy)
  CG_EPI_RAW = 1,     // acc -> fp32 (fc0 pre-activations)
  CG_EPI_DGRAD = 2,   // acc * (mask[row, n] > 0) -> BF16 planes (gradient maps)
  CG_EPI_WGRAD = 3,   // acc -> fp32 weight gradient, plain store or atomic accumulation (split-K)
};
// ACT / DGRAD tiles hand their fp32 sums to the epilogue warpgroup through a 128 x umma_n fp32 buffer in shared memory (carved
// out of the problem's ring budget) and the MMA warps go on to the next tile; RAW / WGRAD tiles (plain stores or red.adds, and
// the conv2 wgrad's 108 KB stages leave no room for a buffer) are finished in place by the MMA warps.  Only the epilogue
// warpgroup signals dependency counters, so only ACT / DGRAD problems may be wired as producers.
__host__ __device__ constexpr bool cg_epi_handoff(int epi) { return epi == CG_EPI_ACT || epi == CG_EPI_DGRAD; }
__host__ __device__ constexpr int cg_acc_bytes(int umma_n) { return 128 * umma_n * 4; }

struct CgLoad {
  int map;            // index of the tensor map (all planes of the tensor: plane = outermost dimension)
  int rank;           // tensor-map rank including the plane dimension (3..5)
  int box_bytes;      // bytes one plane of the box occupies (host-side check)
  int smem_off;       // byte offset of the plane-0 box inside a stage (A boxes below b_off, B boxes from b_off on)
  int plane_stride;   // bytes between the plane copies of the box inside the stage (filled by cg_finalize: a_pstride | b_pstride)
  int plane_box;      // 1: the box spans every plane -> one instruction per chunk, planes land box_bytes apart (== plane_stride);
                      // 0: one instruction per plane (plane = last coordinate)
  int c0[5];          // box start coordinates: c0 + tm*d_tm + tn*d_tn + c1*d_c1 + c2*d_c2 (+ tm_tab)
  int d_tm[5], d_tn[5], d_c1[5], d_c2[5];
};

struct CgProblem {
  // ---- tile grid: tile -> (split, tm, tn); K-chunk c = c1 * n2 + c2
  int tile_start, tiles_m, tiles_n, splits;
  int chunks, n2;
  // ---- operand fetch
  int nloads, planes;
  int a_pstride, b_pstride;   // stage layout: [A plane 0 | A plane 1 | ..][B plane 0 | B plane 1 | ..]; bytes of one A / B plane
  int tx_bytes;               // bytes all boxes of one stage deliver (planes x sum of box bytes)
  int slot_bytes, nstages;    // stage ring geometry of THIS problem (cg_finalize): the problems of a launch share the ring's bytes, not
                              // its partition -- the ring is drained when the partition changes.  The handoff buffer of an ACT / DGRAD
                              // problem follows its ring (byte nstages * slot_bytes)
  CgLoad ld[CG_MAX_LOADS];
  const int* tm_tab;          // optional [tiles_m][CG_MAX_LOADS][2]: extra offsets of coordinates 1 and 2 per (tm, load)
  // ---- MMA
  int mn_major;               // 0: K-major A and B (rows = M|N, 128 B of K); 1: MN-major (rows = K, 128 B of M|N)
  unsigned long long a_desc, b_desc;  // shared-memory descriptor bits of the A / B operand except the start address (cg_desc_bits:
                                      // swizzle span, LBO, SBO); B is always 128B-swizzled, A's rows may be 64 B (conv1, one channel)
  int a_moff;                 // byte offset of the second warpgroup's 64 rows of A inside the A region
  int ksteps;                 // wgmma K = 16 steps per chunk (a template parameter of the kernel's mainloop: part of the shape key)
  int a_off, b_off;           // region offsets inside a stage (b_off = planes * a_pstride)
  int a_kstep, b_kstep;       // descriptor start-address advance per k-step (bytes)
  int a_kstep2;               // A's advance per PAIR of k-steps (2 a_kstep, or the next box when a box row holds two k16 slices)
  int a_lbo, b_lbo;           // MN-major: byte stride between 64-element atoms along M|N
  int umma_n;                 // tile width: 32, 64 or 128 (the widths cg_kernel is instantiated for)
  int nprod;                  // products per k-step: 1 (hi*hi), 3 (+hi*lo, lo*hi), 6 (+mid terms of the 3-plane split), one MMA
                              // each: A_p x B_q into accumulator group p + q, so group g collects the products of order 2^(-8g)
                              // (planes * umma_n <= 256 accumulator columns)
  // ---- epilogue
  int epi;
  int rows_tile;              // real rows of a full tile (<= 128)
  int lim_rows;               // tm * rows_tile + r < lim_rows
  int d0, d1;                 // r -> i0 = r % d0, i1 = (r / d0) % d1, i2 = r / (d0 * d1)
  long long o_tm; int o0, o1, o2; long long o_base;    // output element offset of (tm, r)
  int rgrp_rows;              // > 0: row r also adds rgrp_off[r / rgrp_rows] (conv1 wgrad: one base offset per M atom)
  int rgrp_off[8];
  int lim_i0;                 // > 0: rows with i0 >= lim_i0 are not stored (junk columns of conv1, padded channels of its wgrad)
  int tm_sub;                 // > 1 (ACT / DGRAD): row-tile tm is band tm % tm_sub of block tm / tm_sub -- its output starts at
  long long o_sub;            //   (tm / tm_sub) * o_tm + (tm % tm_sub) * o_sub, and rows with (tm % tm_sub) * d1 + i1 >= lim_i1
  int lim_i1;                 //   are not stored (conv1: two 8 x 16 bands of a sample's 15 x 15 output map)
  long long m_tm; int m0, m1, m2; long long m_base;    // mask element offset of (tm, r)
  int n_valid;                // columns < n_valid are stored (N of the problem)
  int grp_stride;             // element distance between consecutive 32-column groups of the output (32 = contiguous)
  int grp_tab;                // 1: per-group output / mask offsets and row limits come from the tables below (conv2 dgrad: one
                              //    accumulator column group per output-parity class)
  int grp_off[8], grp_moff[8], grp_lim0[8], grp_lim1[8];
  int out_planes;             // planes written by ACT / DGRAD
  uint16_t* out_p[CG_MAX_PLANES];
  float* out_f;               // fp32 output (RAW / WGRAD; optional extra copy for ACT), same offsets, ld = o0-based
  long long f_tm; int f0;     // fp32 copy: offset = tm * f_tm + r * f0 + col   (ACT extra copy only; 0 = none)
  const float* bias;          // [N]
  int bias_grp;               // element distance between the bias blocks of consecutive 32-column groups (32 = contiguous)
  long long f_grp;            // same for the fp32 copy
  const uint16_t* mask;       // hi plane of the forward activation (DGRAD)
  float* colsum;              // DGRAD: bias gradient of the layer = column sums of the masked gradient map, accumulated (red.add) from the
  int colsum_mask;            //        fp32 accumulators: colsum[(column) & colsum_mask]   (nullptr: none)
  int atomic;                 // WGRAD: 1 = red.add (split-K or shared output), 0 = store
  float scale;                // WGRAD: multiply before accumulation (1 = none)
  // ---- dependencies between the problems of ONE launch (fused layers).  Tiles are dealt to the CTAs in increasing order and
  //      every CTA of the grid is resident, so a tile may wait for lower-numbered tiles of an earlier problem: the producers of
  //      tile tm spin until the row-tiles [tm * dep_rows / dep_rows_tile, ((tm + 1) * dep_rows - 1) / dep_rows_tile] of the
  //      producing problem have each collected dep_expect arrivals (x CG_EPI_WARPS: one per epilogue warp and (tn, split) tile), then order the
  //      generic-proxy stores they observed before their own async-proxy (TMA) reads.
  int* done_ctr;              // arrival counters of THIS problem, one per tm (nullptr: nobody waits on it); zeroed before the launch
  const int* dep_ctr;         // counters of the producing problem (nullptr: no dependency)
  int dep_rows, dep_rows_tile, dep_tiles, dep_expect;
  // ---- split-K with in-kernel finalisation (ACT problems with splits > 1; the late layers have too few tiles for 132 SMs): every
  //      split tile adds its fp32 partial sums into ws[tile][128][umma_n] (red.add), then each epilogue warp bumps its own arrival
  //      counter of the tile; the warp that arrives LAST reads the sums back, clears them for the next step, and runs the normal
  //      bias / ReLU / plane-split / store path (and alone signals done_ctr)
  float* ws;                  // nullptr: splits are plain (RAW / WGRAD atomics)
  int* ws_cnt;                // [tiles_m * tiles_n][CG_EPI_WARPS]
  // ---- data parallel (N > 1): a weight gradient that is FINAL when its tile is stored (no split-K) is also pushed, float4 by float4,
  //      into the receive arena of the rank that owns that part of the gradient arena (optim.cu: dp_optim_kernel) -- 80 % of the
  //      gradient bytes leave while the backward pass is still running
  float* dp_recv[8];          // receive arenas (nullptr entries: none)
  const float* dp_gbase;      // base of the local gradient arena (owner of float4 i4 = i4 / dp_per4)
  int dp_rank, dp_n, dp_per4;
  int dep_by_chunk;           // 1: the rows are indexed by the tile's K-chunk range [c_begin, c_end) instead of its tm (weight gradients)
};

struct CgGroup {               // one launch
  CgProblem host[CG_MAX_PROBLEMS];
  int n = 0;
  int total_tiles = 0;
  int slot_bytes = 0, nstages = 0, ring_bytes = 0;     // largest slot / most stages of any problem; bytes of the ring (with the handoff buffer)
  const char* name = "";
  double flops = 0;
};

// encodes a BF16 tiled tensor map (zero OOB fill, SWIZZLE_<swizzle>B: 128 or 64, the bytes of the box's innermost dimension);
// dims/box innermost first, strides in BYTES for dims 1..rank-1
int cg_encode_map(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                  const uint32_t* elem_strides, int swizzle = 128);
// descriptor bits of a wgmma shared-memory operand (everything but the start address) whose rows are `swizzle` bytes (128 or 64)
// swizzled: K-major (rows = M|N; SBO = 8 rows, LBO unused) or MN-major (rows = K; SBO = 8 rows, LBO = stride between atoms
// of swizzle / 2 elements along M|N)
unsigned long long cg_desc_bits(int swizzle, bool mn_major, int lbo);
// finalises tile_start / total_tiles / ring geometry of a group (host side)
int cg_finalize(CgGroup& g, int smem_budget);
cudaError_t cg_launch(const CgGroup& g, const CUtensorMap* dev_maps, int num_sms, cudaStream_t s, bool pdl, int debug_flags);
int cg_smem_limit();
// cg_kernel is compiled for a fixed set of (tile width, products per k-step, MN-major, k-steps per chunk) shapes; a problem of
// any other shape is rejected when its group is built
__host__ __device__ constexpr int cg_shape_key(int umma_n, int nprod, bool mn_major, int ksteps) {
  return ksteps * 8192 + umma_n * 16 + nprod * 2 + (mn_major ? 1 : 0);
}
bool cg_shape_supported(int umma_n, int nprod, bool mn_major, int ksteps);

}  // namespace b2g
