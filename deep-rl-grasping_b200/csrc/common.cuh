// Shared declarations of libb200grasp (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

namespace b2g {

// ---------------------------------------------------------------------------------------------
// Programmatic dependent launch: a kernel launched through launch_pdl() may start (smem carve-up,
// barrier init) while its predecessor on the stream is still running; it must call
// pdl_wait() before touching global memory, and pdl_trigger() lets ITS successor start early.
// ---------------------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, bool pdl, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
#endif
bool pdl_enabled();   // sac.cu: B2G_PDL != 0

// ---------------------------------------------------------------------------------------------
// Gather-GEMM problem descriptor.  One engine serves every dense contraction on the path:
//   C[cM[m] + cN[n]]  (=|+=)  epi( sum_r  A[aM[m] + aR[r]] * B[bR[r] + bN[n]] )
// The offset tables (built once on the host, resident in HBM/L2) encode im2col for the forward
// convolutions, the transposed/patch-major views for wgrad, and the parity-class gathers over
// zero-bordered gradient maps for dgrad, so no im2col matrix is ever materialised.
// ---------------------------------------------------------------------------------------------
enum GemmFlags : int {
  GG_A_RVEC = 1 << 0,     // A offsets contiguous along r in aligned groups of 4 (else along m)
  GG_B_RVEC = 1 << 1,     // B offsets contiguous along r in aligned groups of 4 (else along n)
  GG_EPI_BIAS_RELU = 1 << 2,
  GG_EPI_MASK = 1 << 3,   // C = acc * (mask[kM[m] + kN[n]] > 0)
  GG_EPI_ATOMIC = 1 << 4, // split-R accumulate into pre-zeroed C
  GG_COLSUM = 1 << 5,     // colsum[n] += sum_r B(r, n)   (bias gradients; tile_m == 0 only)
  GG_PLANES = 1 << 6,     // operands come pre-split as BF16 hi/lo planes (A_hi.., B_hi..), copied by cp.async
  GG_A_ALIGN4 = 1 << 7,   // plane A rows are only 8-byte aligned (conv1 with one image channel)
  GG_EPI_BIAS = 1 << 10,  // C = acc + bias[n] (no activation; output layers)
  GG_EPI_SCALE = 1 << 11, // C = acc * alpha (after mask)
  GG_A_SCALAR = 1 << 12,  // fp32 engine, with GG_A_RVEC: no 4-element contiguity along r -> element-wise gather (1-channel convs);
                          // gg_simt_launch_ext also without GG_A_RVEC (no contiguity along m)
  GG_A_ROWLANES = 1 << 14, // planes K-major producer: lanes walk 8 consecutive rows of one 16-byte column group (conv1: adjacent
                           // output pixels overlap in the image, so a warp copy touches 4-8 lines instead of 32)
  GG_EPI_BIAS_LRELU = 1 << 13, // C = leaky_relu(acc + bias[n], slope alpha)   (Keras LeakyReLU; encoder.cu)
  GG_MN_MAJOR = 1 << 9,   // planes mode, wgrad: both operands contiguous along their M / N index -> MN-major wgmma tiles
  GG_CN_AFFINE4 = 1 << 8, // host-verified: cN / kN contiguous inside aligned 4-column groups, outputs 16-byte aligned
  GG_EPI_LRELU_GRAD = 1 << 15, // gg_simt_launch_ext: C = acc * g(mask[kM[m] + kN[n]]), g = 1 / alpha / 0 for a post-LeakyReLU value
                               // > 0 / < 0 / == 0 (Keras' relu(x) - alpha * relu(-x) has gradient 0 at x = 0)
  GG_EPI_BIAS_TANH = 1 << 16,  // gg_simt_launch_tanh: C = tanh(acc + bias[n])
  GG_EPI_TANH_GRAD = 1 << 17,  // gg_simt_launch_tanh: C = acc * (1 - y^2), y = mask[kM[m] + kN[n]] a stored tanh output
  GG_ACC64 = 1 << 18,          // gg_tc_launch: the auto-encoder training instantiations (GG_EPI_BIAS_LRELU, GG_EPI_LRELU_GRAD, and
                               // GG_EPI_ATOMIC / GG_COLSUM adding fp32 split partials into double arrays behind C / colsum)
};

struct GemmDesc {
  const float* A;
  const float* B;
  float* C;
  const int* aM; const int* aR;
  const int* bR; const int* bN;
  const int* cM; const int* cN;
  const int* kM; const int* kN;
  const float* bias;
  const float* mask;
  float* colsum;
  // BF16 hi/lo planes (same element offsets as the fp32 tensors; B planes may use their own tables)
  const uint16_t* A_hi; const uint16_t* A_lo;
  const uint16_t* B_hi; const uint16_t* B_lo;
  const int* bR_p; const int* bN_p;
  uint16_t* C_hi; uint16_t* C_lo;      // optional plane copy of the output (feeds the next contraction)
  float alpha;                         // GG_EPI_SCALE
  int M, N, R;
  int flags;
  int splitR;
  int tiles_m, tiles_n;
  int tile_start;   // first flattened CTA index of this problem inside a grouped launch
  int tile_count;
  int col_id;       // wgmma engine: identity of (cN, kN, bias, N); equal ids share the staged column tables
};

struct GemmGroup {          // one grouped launch
  std::string name;
  std::vector<GemmDesc> host;
  GemmDesc* dev = nullptr;
  int total_tiles = 0;
  double flops = 0;
  bool tc = false;          // run on the wgmma engine
};

// engines (gg_simt.cu / gg_tc.cu)
void gg_simt_launch(const GemmDesc* dev_descs, int ndesc, int total_tiles, cudaStream_t s);
// the same engine with GG_EPI_LRELU_GRAD and m-contiguous GG_A_SCALAR gathers, summing in double, with GG_EPI_ATOMIC /
// GG_COLSUM accumulating into double arrays behind C / colsum (auto-encoder training, autoencoder.cu)
void gg_simt_launch_ext(const GemmDesc* dev_descs, int ndesc, int total_tiles, cudaStream_t s);
// the plain fp32 engine with the tanh epilogues GG_EPI_BIAS_TANH and GG_EPI_TANH_GRAD (PPO's MLP, ppo.cu)
void gg_simt_launch_tanh(const GemmDesc* dev_descs, int ndesc, int total_tiles, cudaStream_t s);
constexpr int GG_SIMT_BM = 64, GG_SIMT_BN = 64, GG_SIMT_BK = 16;
// wgmma engine: 128 x 64 output tile, 64-wide r-chunks; x3 != 0 -> BF16 hi/lo split (3 MMAs)
cudaError_t gg_tc_launch(const GemmDesc* host_descs, int ndesc, int total_tiles, int mode_flags, int x3, int num_sms, cudaStream_t s);
constexpr int GG_TC_MAX_DESCS = 16;
int gg_tc_smem_bytes();
// sets the shared-memory opt-in of the GG_ACC64 instantiations (before a graph capture launches them)
cudaError_t gg_tc_acc64_init();
constexpr int GG_TC_BM = 128, GG_TC_BN = 64, GG_TC_BK = 64;

// ---------------------------------------------------------------------------------------------
// head "tail" kernel (tail.cu): everything after the fc0 contractions, per sample
// ---------------------------------------------------------------------------------------------
struct HeadW {           // pointers into the parameter arena for one MLP head
  const float* b0;       // fc0 bias [H]
  const float* k1;       // fc1 kernel [H,H]
  const float* b1;       // fc1 bias [H]
  const float* ko;       // output kernel [H, n_out]
  const float* bo;       // output bias [n_out]
  const float* k0;       // fc0 kernel [in, H] (qf heads: rows feat_dim.. are the action rows)
};
struct HeadG {           // matching gradient-arena pointers (small tensors accumulated by the tail)
  float* b1; float* ko; float* bo;
};

struct TailArgs {
  int B, H, A, feat_dim;
  float gamma, target_entropy;
  int grad_scale_B;            // divide means by this batch size (local batch)
  // fc0 pre-activations (no bias) [B,H] each
  const float* z0_pi; const float* z0_vf; const float* z0_q1; const float* z0_q2; const float* z0_vt;
  int z0v_ld;                  // row stride of z0_vf / z0_q1 / z0_q2 (H, or 3H when the three heads share one [B,3H] block)
  HeadW pi, vf, q1, q2, vt;
  const float* ksig; const float* bsig;      // pi: dense_1 (log_std) kernel/bias; pi.ko/bo = dense (mu)
  HeadG g_pi, g_vf, g_q1, g_q2;
  float* g_ksig; float* g_bsig;
  const float* log_alpha; float* g_log_alpha;
  const float* act;  int act_stride;         // replay actions (inside F_V rows)
  const float* eps;                          // [B,A]
  const float* rew; const float* done;       // normalised reward, done [B]
  // saved for the engine: post-ReLU fc0 activations and gradients
  float* a0_pi; float* a0_vf; float* a0_q1; float* a0_q2;   // [B,H]
  float* dz1_pi; float* dz1_vf; float* dz1_q1; float* dz1_q2; // [B,H]
  float* dz0_pi;                               // [B,H]
  float* dz0_v3;                               // [B,3H] = vf | q1 | q2
  uint16_t* dz0_pi_p[2]; uint16_t* dz0_v3_p[2];  // optional BF16 hi / lo planes of the same (engine v2 operands)
  float* per_sample;                           // 7 x [B]: q1,q2,v,logp,v_targ,q1_pi,q2_pi
  float* pi_out;                               // [B,A]
  float* metrics;                              // accumulators (see MET_* in sac.cu)
};
cudaError_t tail_launch(const TailArgs& a, cudaStream_t s, bool pdl);   // pdl: may start while its predecessor drains

// Weight gradients of the head MLPs (fc0 / fc1 kernels and biases of pi, vf, qf1, qf2) in fp32 on the CUDA cores: 76 MFLOP
// of [B]-deep reductions, too small for a tensor-engine launch (which would also hold every SM while it runs).
struct HeadsWgradArgs {
  const float* X0[4];     // fc0 inputs: feature rows [B][x0_ld] (pi: F_pi; vf, qf1, qf2: F_values incl. the action columns)
  const float* dz0[4];    // fc0 pre-activation gradients [B][dz0_ld[q]] (column offset applied)
  const float* a0[4];     // fc0 activations [B][H]
  const float* dz1[4];    // fc1 pre-activation gradients [B][H]
  float* g_k0[4]; float* g_b0[4]; float* g_k1[4]; float* g_b1[4];
  int M0[4];              // fc0 input width of head q (kernel rows)
  int dz0_ld[4];
  int x0_ld, B;
  int H;                  // head width (a multiple of 64)
};
void heads_wgrad_launch(const HeadsWgradArgs& a, cudaStream_t s);
// policy inference tail: tanh(mu) or tanh(mu + eps*std) for the first n rows of z0_pi
cudaError_t act_launch(const TailArgs& t, int n, int deterministic, float* act_out, cudaStream_t s);

enum Metric : int {
  MET_POLICY_LOSS = 0, MET_QF1_LOSS, MET_QF2_LOSS, MET_VALUE_LOSS, MET_ENT_COEF_LOSS, MET_ENTROPY,
  MET_MEAN_Q1, MET_MEAN_Q2, MET_MEAN_V, MET_MEAN_LOGP, MET_GN_PI, MET_GN_VALUES, MET_COUNT = 16
};

// ---------------------------------------------------------------------------------------------
// optimiser (optim.cu): 3x TF-Adam + Polyak over the flat arenas, one launch
// ---------------------------------------------------------------------------------------------
struct OptimArgs {
  float* P; float* Mo; float* Vo; const float* G;   // trainable arenas
  float* T;                                          // target block (same relative layout as values block)
  int n_pi, n_values, n_ent;                         // padded segment lengths: [pi | values | ent]
  int n_target;                                      // padded length of the target block
  const double* step_consts;                         // [3] lr_t per optimiser (device, written by prep kernel)
  float tau;
  float grad_scale;                                  // 1/nranks after a sum all-reduce
  float* metrics;                                    // MET_GN_* accumulators
  int apply;                                         // 0 = only grad norms
  long long* bump_counter;                           // rng step counter advanced once per step (nullptr: prep did it)
  int r_lo[2], r_hi[2];                              // optional: update only arena ranges [r_lo, r_hi) (floats, multiples of 4);
                                                     // all zero = the whole arena
};
void optim_launch(const OptimArgs& a, cudaStream_t s);

// Data-parallel optimiser step over NVLink peer memory (optim.cu): reduce-scatter of the gradient arena, Adam / Polyak on the
// owned shard and all-gather of the updated parameters in ONE kernel.  Rank r owns the r-th 1/N of the arena: every rank pushes
// that slice of its gradients into r's receive arena (peer stores), r sums the N copies in fixed rank order (replicas stay
// bit-identical), updates its slice of P / m / v (the moments exist only on the owner) and stores the new parameters -- and the
// Polyak-averaged target slice -- into every rank's arena, again through peer stores.  Ranks meet twice through epoch flags in each other's memory (release /
// acquire at system scope): "my gradients are final" before the loads, "my slice is written everywhere" before the kernel ends.
constexpr int DP_MAX_RANKS = 8;
struct DpArgs {
  OptimArgs o;                         // local arenas, step sizes, metrics
  int rank, nranks;
  float* R_peer[DP_MAX_RANKS];         // receive arena of every rank: [src rank][slice] floats (slices pushed by their producers)
  float* P_peer[DP_MAX_RANKS];         // parameter arena of every rank
  int* x_peer[DP_MAX_RANKS];           // exchange block of every rank: int flags[2][8] (G ready, slice written), float part[8][2], loss[8][16]
  int skip_lo4[2], skip_hi4[2];        // float4 ranges of the arena whose slices were already pushed by the backward epilogues
  const long long* counters;           // counters[3] = optimiser step = flag epoch
  int* sync;                           // local: [0], [1] CTA arrival counters, [2..3] squared-norm accumulators (as float), [8..] bring-up stamps
};
void dp_optim_launch(const DpArgs& a, int ctas, cudaStream_t s);

// weights -> BF16 hi/lo planes, original [R,N] layout and transposed [N,R] (optim.cu)
struct PlaneJob {
  const float* src;            // [R, N] row-major fp32 (TF layout: HWIO filters flattened, dense [in,out])
  uint16_t* hi; uint16_t* lo;  // [R, N] planes (may be null)
  uint16_t* hiT; uint16_t* loT;// [N, R] planes (may be null)
  int R, N;
  int tile_start;              // first 32x32 tile of this job in the flattened launch
};
void planes_launch(const PlaneJob* dev_jobs, int njobs, int total_tiles, cudaStream_t s);
// bias gradients: dst[n] += sum over rows of src[row_off[m] + n]  (optim.cu)
struct ColsumJob { const float* src; const int* row_off; float* dst; int rows, N; int cta_start; };
void colsum_launch(const ColsumJob* dev_jobs, int njobs, int total_ctas, cudaStream_t s);

struct PrepArgs {          // 1-CTA kernel at the head of every step
  long long* counters;     // [0..2] Adam t per optimiser, [3] n_updates, [4] rng step counter
  double* step_consts;     // lr_t x3
  const float* lr;         // device scalar
  float* metrics;          // zeroed
  int* indices; float* eps;// generated when gen != 0
  int B, A; const long long* replay_size;   // nullptr -> counters[5]
  long long ring_cap;      // > 0: slots are (counters[6] + u) % ring_cap (replay that lost transitions early starts mid-ring)
  unsigned long long seed; int gen; int apply;
  int defer_bump;          // 1: the rng step counter [4] is advanced by the optimiser kernel at the end of the step
  int skip_indices;        // 1: the gather kernel draws the replay slots itself (same Philox stream)
};
void prep_launch(const PrepArgs& a, cudaStream_t s);

// ---------------------------------------------------------------------------------------------
// replay row compaction, gather + VecNormalize + /255 (replay.cu)
// ---------------------------------------------------------------------------------------------
// full observations [n][HW][Cfull] -> compact rows (first_row + i) % wrap of dst: image planes [HW][Ci] | value at pixel [0,0]
// of plane Ci (Cfull == Ci + 1, the augmented extractor's direct feature; 0 when Cfull == Ci) | 3 zero pads
void compact_rows(const float* src_full, float* dst, long long first_row, long long wrap, int n, int HW, int Ci, int Cfull,
                  cudaStream_t s);

// How a replay frame stores one compact row of Ec floats: npx image elements [HW][Ci] (NHWC), then a tail of Ec - npx floats
// (CNN: the actuator value and 3 pads; MLP: npx = 0 and the tail is the whole observation).  Image channel c lives in the
// pixel's uint8 block when ch[c] >= 0 (byte ch[c] of [HW][n8] at offset 0) and in its fp32 block otherwise (float -1 - ch[c] of
// [HW][n32] at byte f32_off).  n8 == 0 is the plain fp32 compact row (ch unused).
struct FrameFmt {
  int n8, n32;
  int f32_off, tail;         // byte offsets of the fp32 image block and of the tail
  signed char ch[8];
};
#ifdef __CUDACC__
// element e of the compact row stored in frame f (decoded values are exactly the values the caller passed); the host decodes
// a frame it read back the same way (TransitionReplay::get)
__host__ __device__ __forceinline__ float frame_elem(const unsigned char* __restrict__ f, const FrameFmt& m, int npx, int Ci, int e) {
  if (e >= npx) return reinterpret_cast<const float*>(f + m.tail)[e - npx];
  if (m.n8 == 0) return reinterpret_cast<const float*>(f)[e];
  const int pix = e / Ci, k = m.ch[e - pix * Ci];
  return k >= 0 ? (float)f[pix * m.n8 + k] : reinterpret_cast<const float*>(f + m.f32_off)[pix * m.n32 - 1 - k];
}
// image elements [e, e + 4) (e % 4 == 0): one 128-bit load for fp32 frames
__device__ __forceinline__ float4 frame_load4(const unsigned char* __restrict__ f, const FrameFmt& m, int npx, int Ci, int e) {
  if (m.n8 == 0) return *reinterpret_cast<const float4*>(f + 4 * (size_t)e);
  return make_float4(frame_elem(f, m, npx, Ci, e), frame_elem(f, m, npx, Ci, e + 1), frame_elem(f, m, npx, Ci, e + 2),
                     frame_elem(f, m, npx, Ci, e + 3));
}
#endif

// Replay frame pool writes (replay.cu).  frame_check: flags[i] bit 0 = compact row c_obs[i] equals frame prev[i] bit for bit
// (prev[i] < 0: no candidate), bit 1 = a value of c_obs[i] or c_next[i] in a uint8 channel is not an integer in [0, 255].
// frame_commit: c_obs[i] -> frame plan[i] when plan[m + i] != 0, c_next[i] -> frame plan[2m + i], and transition slot
// (first + i) % cap records both frame indices.  plan == nullptr: row i takes the new frames fid0 + 2i, fid0 + 2i + 1
// (mod fcap), which needs no upload when no frame is shared.
struct FrameIo {
  const float* c_obs; const float* c_next;   // compact rows [m][Ec]
  unsigned char* frames; long long frame_bytes;
  FrameFmt fmt; int npx, Ci, Ec;
};
void frame_check_launch(const FrameIo& io, const int* prev, int* flags, int m, cudaStream_t s);
void frame_commit_launch(const FrameIo& io, const int* plan, long long fid0, long long fcap, int m, int* r_ofr, int* r_nfr,
                         long long first, long long cap, cudaStream_t s);

struct GatherArgs {
  const float* obs; const float* next_obs; const float* act; const float* rew; const float* done; // replay or staged batch
  // replay frame pool: when obs_frame != nullptr, sample slot s reads frames obs_frame[s] / next_frame[s] instead of obs / next_obs
  const unsigned char* frames; long long frame_bytes; const int* obs_frame; const int* next_frame;
  FrameFmt fmt;              // layout of the rows read (frames, or the fp32 compact rows of obs / next_obs)
  long long ring_cap;        // in-kernel slot draw: slot = (rng_counters[6] + u) % ring_cap, u uniform in [0, size)
  const int* indices;        // [B] slot per sample (nullptr: identity)
  const double* mean; const double* var; // [row elems]; var[] holds 1/sqrt(var+eps)
  const double* normc;       // device: {1/sqrt(ret_var+eps), clip_obs, clip_rew, norm_obs, norm_rew}
  int B, H, W, Cimg;         // CNN: compact rows of an [H,W,Cimg] image (replay.cu); MLP: H = 0, W = obs_dim
  float scale;               // 255 for CNN, 1 for MLP
  float* x_obs; float* x_next;   // CNN: [B,H,W,Cimg] image planes (scaled)
  uint16_t* x_obs_hi; uint16_t* x_obs_lo; uint16_t* x_next_hi; uint16_t* x_next_lo;   // optional BF16 planes of x
  float* F_pi; float* F_v; float* F_t; int FS; int feat_col; // feature rows: direct feature -> col feat_col; MLP: whole obs -> cols 0..
  int act_col;               // CNN: feature-row column of the first replay action (feat_col < 0: no direct feature)
  float* rew_out; float* done_out; int n_act;
  // in-kernel slot draw (indices == nullptr && rng_counters != nullptr): Philox stream 0 of prep_kernel, same values
  const long long* rng_counters;   // [4] = rng step, [5] = replay size, [6] = first live slot (ring_cap > 0)
  unsigned long long seed;
  int* indices_out;                // optional record of the drawn slots
};
void gather_launch(const GatherArgs& a, cudaStream_t s);

// VecNormalize obs_rms merge (obsnorm.cu): the n frames a[i] (b[i] where done[i] != 0 when b != nullptr) -> float64 mean / var
// [E] by RunningMeanStd.update_from_moments with the prior count, then the gather's table d_mean / d_istd = 1/sqrt(var + eps).
// Table layout: Cfull > 0 = CNN compact rows of [HW][Cfull] frames (image planes, then the actuator value at index npx);
// Cfull == 0 = flat, entry e for element e.  n == 0 only derives the table.
void obs_rms_update_launch(const float* a, const float* b, const float* done, int n, int E, double count, double eps, double* mean,
                           double* var, double* d_mean, double* d_istd, int Cfull, int npx, cudaStream_t s);

// Philox4x32-10 (counter-based RNG shared by prep_kernel and the in-kernel replay slot draw)
#ifdef __CUDACC__
__device__ __forceinline__ void philox_round(uint4& c, uint2& k) {
  const unsigned hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
  const unsigned hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
  c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  k.x += 0x9E3779B9u; k.y += 0xBB67AE85u;
}
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int i = 0; i < 10; ++i) philox_round(c, k);
  return c;
}
// replay slot of sample b at rng step `step`: element (b & 3) of block b >> 2 of stream 0, scaled to [0, rsz)
__device__ __forceinline__ int philox_slot(unsigned long long seed, unsigned long long step, int b, unsigned long long rsz) {
  const uint4 r = philox4x32_10(make_uint4((unsigned)step, (unsigned)(step >> 32), (unsigned)(b >> 2), 0u),
                                make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
  const unsigned v = (b & 3) == 0 ? r.x : (b & 3) == 1 ? r.y : (b & 3) == 2 ? r.z : r.w;
  return (int)(((unsigned long long)v * rsz) >> 32);
}
// u-th live slot of a ring whose live range starts at slot base (u < cap)
__device__ __forceinline__ int ring_slot(long long base, int u, long long cap) {
  const long long s = base + u;
  return (int)(s >= cap ? s - cap : s);
}
#endif

}  // namespace b2g
