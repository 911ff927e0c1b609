// The transition replay of the SAC, BDQ and DQN learners, with proportional prioritised replay on the device (per.cu).
//
// [SB2] common/buffers.py PrioritizedReplayBuffer over common/segment_tree.py (Schaul et al. 2016), with the sum / min
// segment trees resident in HBM: leaves C..2C-1 (C = capacity rounded up to a power of two), node i = f(2i, 2i+1).  Sums are
// kept in float64 like the Python floats of the reference.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <functional>
#include <vector>

#include "../../include/b200grasp.h"
#include "common.cuh"
#include "frame_ring.cuh"
#include "state.cuh"

namespace b2g {

struct PerArgs {
  double* tsum; double* tmin; long long C;
  float* max_prio;                  // running max of the raw priorities (new transitions enter with it)
  const long long* counters;        // [4] rng step, [5] replay size, [6] first live slot (ring_cap > 0)
  long long ring_cap;               // > 0: a replay with frames, whose live window may start mid-ring and skip evicted slots
  unsigned long long seed;
  int B; float alpha, eps; const float* beta;
  int* indices; float* weights; float* prio_out;
  const float* td; int D;
};

// One CTA of round32(B) threads: draws B slots proportionally to priority (find_prefixsum_idx descent, Philox stream 2 at
// counters[4]) and their importance-sampling weights (p_i size)^-beta / max_w.  B <= 1024.
void per_sample_launch(const PerArgs& a, cudaStream_t s);
// One CTA of round32(n) threads (n <= 1024): writes n leaves and repairs their ancestors.  The leaves are slots[i], or
// (first_slot + i) % cap when slots == nullptr.  from_td == 1: raw priority sum_d |td[i * D + d]| + eps (also written to
// prio_out and folded into max_prio); 0: the running max_prio.  Leaf value raw^alpha.  from_td == 2: the slots left the replay
// (evicted early): sum 0, min +inf.
void per_write_launch(const PerArgs& a, const int* slots, long long first_slot, long long cap, int n, int from_td, cudaStream_t s);
// Empty trees of n2 = 2C nodes (sum 0, min +inf) and max_prio = 1.
void per_init_launch(double* tsum, double* tmin, long long n2, float* max_prio, cudaStream_t s);

// Caller rows src [m][E] (host or device) -> the compact rows dst [m][Ec] of the add staging, enqueued on the replay's stream
using RowLoader = std::function<int(const float* src, float* dst, int m)>;

// Ring of cap transitions (obs [E], action [A], reward, done as float rows) and, with prioritised replay, its trees.  Row i of
// every ring is transition i; pos is the next row written, size the number of live rows.
//
// With frames (frame_cap > 0): obs and next_obs live in a pool of frame_cap frames, and slot s names its two frames in
// r_ofr[s] / r_nfr[s] (FrameRing's numbering and eviction, frame_check / frame_commit).  A frame stores one compact row of
// io.Ec floats in the layout io describes: SAC's image rows, optionally with 8-bit planes, or the plain fp32 rows of BDQ and
// DQN (plain_frames).  Every next_obs takes a new frame; row i's obs shares the previous call's next_obs frame of row i when
// the two are bit-equal (add) or by construction (add_linked from the observe path).  The live window is [tail, tail + size)
// mod cap (counters[6] = its first slot once transitions went early); evicted slots leave the prioritised-replay trees.
struct TransitionReplay {
  float *obs = nullptr, *next = nullptr, *act = nullptr, *rew = nullptr, *done = nullptr;
  int64_t cap = 0, size = 0, pos = 0;
  int E = 0, A = 0;                                     // E: floats of a caller's observation
  bool per = false;
  float alpha = 0.f, eps = 0.f;                         // priority exponent and the epsilon added to |TD|
  double *t_sum = nullptr, *t_min = nullptr;
  long long per_C = 0;
  float *max_prio = nullptr, *beta = nullptr, *prio_out = nullptr;   // prio_out: [B] priorities of the last sampled step
  long long* h_rc = nullptr;                            // pinned: replay size, first live slot -> counters[5..6]
  // frames (frame_cap > 0 only)
  FrameRing ring;
  FrameIo io{};                                         // the frame layout and pool (c_obs / c_next unset)
  int *r_ofr = nullptr, *r_nfr = nullptr;
  float *c_obs = nullptr, *c_next = nullptr;            // add's staging: compact rows [stage_rows][io.Ec]
  int *d_plan = nullptr, *h_plan = nullptr;             // [4][stage_rows]: frame plan (3 rows) + check flags; h_plan pinned
  int stage_rows = 0;                                   // rows per commit launch
  const char* frames_name = "frame_capacity (replay_frames)";   // the frame budget as the handle's callers name it, in refusals

  // Allocates the rings, and the trees (empty, beta 0.4) when per; B is the batch of a sampled step.  frame_cap > 0: obs and
  // next_obs as frames of `layout` (frame_cap >= cap + 1), commits of up to stage_rows rows.
  int init(std::vector<void*>& allocs, cudaStream_t s, int64_t cap, int E, int A, int B, bool per, float alpha, float eps,
           int64_t frame_cap = 0, const FrameIo& layout = {}, int stage_rows = 0);
  // Frees the pinned staging (the device buffers belong to allocs).
  void release();
  bool framed() const { return io.frames != nullptr; }
  // The prioritised-replay arguments of a sampled step of B rows: draws into indices / weights, new priorities from td [B][D].
  PerArgs per_args(const long long* counters, unsigned long long seed, int B, int* indices, float* weights, const float* td, int D) const;
  // The ring window the uniform draw of prep_kernel reads (0 without frames: slots [0, size))
  long long ring_cap() const { return framed() ? cap : 0; }
  // Points g's replay reads at this replay: obs / next_obs rows or frames through r_ofr / r_nfr, act (with_next), rew, done.
  void gather_args(GatherArgs& g, bool with_next) const;
  // n transitions (host or device rows) at pos, in chunks that end at the ring's end; new rows enter at the running maximum
  // priority.  Then the size goes to counters[5] (and the first live slot to counters[6]) and the stream is drained.  Frames:
  // load (null: a plain copy of io.Ec floats per row) stages each chunk's rows; with 8-bit planes every row is checked before
  // any is stored.
  int add(const float* o, const float* a, const float* r, const float* nx, const float* d, int64_t n, long long* counters, cudaStream_t s,
          const RowLoader& load = nullptr);
  // Frames only: n transitions whose compact rows sit in device memory at c_obs / c_next, act / rew / done host or device.
  // cand[i] >= 0 names a frame that already holds c_obs[i] (shared while it outlives this row's next_obs frame); next_ids[i]
  // receives the frame id of c_next[i].  Enqueued on s, which the caller synchronises before it returns.
  int add_linked(const float* c_obs, const float* c_next, const int64_t* cand, const float* a, const float* r, const float* d, int n,
                 int64_t* next_ids, long long* counters, cudaStream_t s);
  // Rows [first, first + n) (mod cap) enter at the running maximum priority ([SB2] PrioritizedReplayBuffer.add); nothing
  // without per.
  void insert_max_prio(int64_t first, int64_t n, cudaStream_t s) const;
  // pos and size after n more rows
  void advance(int64_t n);
  int set_beta(float beta, int device, cudaStream_t s);
  // b2g_*_get_last_per: slots of the last sampled step (uniform replay too), and with per its weights and new priorities
  int get_last(const int* indices, const float* weights, int B, int32_t* slots, float* w, float* p, int device, cudaStream_t s) const;
  // The stored transition of a live slot (any output may be NULL): obs / next_obs as rows of E floats, or with frames as the
  // compact rows of io.Ec floats their frames hold; frame_ids: its obs / next_obs frames, -1 without frames
  int get(int64_t slot, float* o, float* a, float* r, float* nx, float* d, int32_t* frame_ids, int device, cudaStream_t s) const;
  // b2g_*replay_info
  void info(int64_t* capacity, int64_t* size, int64_t* frame_capacity, int64_t* live_frames, int64_t* bytes, int64_t* evicted_early) const;
  // Without frames: the training-state sections ROBS, RNXT, RACT, RREW, RDON of a replay holding `live` rows (rows [0, live)
  // are the live ones, the rings up to cap for the rest).  With frames: ROFR, RNFR, RACT, RREW, RDON, FRMS (frames [lo, hi) of
  // the pool).
  std::vector<StateSection> state_sections(int64_t live, int64_t lo = 0, int64_t hi = 0) const;
  // The prioritised-replay sections PERT (the trees, empty without per) and PERS (max priority, beta)
  std::vector<StateSection> per_sections() const;
  // The HOST section of a BDQ / DQN training-state file: size, pos, n_updates, eps_bits, then with frames FrameRing::pack().
  std::vector<int64_t> state_host(int64_t n_updates, int64_t eps_bits) const;
  // Reads and checks the HOST section of rd into *hv and (with frames) *ring, the handle unchanged
  int state_host_read(StateReader& rd, std::vector<int64_t>* hv, FrameRing* ring) const;
  // size and pos a file may restore
  bool valid(int64_t size, int64_t pos) const { return size >= 0 && size <= cap && pos >= 0 && pos < cap && (size == cap || pos == size); }

  // add / add_linked, frames: m <= stage_rows transitions whose compact rows sit at c_obs / c_next, planned, committed and their
  // act / rew / done copied, enqueued on s (h_plan must be free: the previous chunk's upload has run)
  int commit(const float* c_obs, const float* c_next, int m, const int64_t* cand, const float* a, const float* r, const float* d,
             int64_t* next_ids, cudaStream_t s);
  // after the last commit of a call: the next call's sharing candidates, size and pos, and counters[5..6]
  int finish(std::vector<int64_t>& next_ids, long long* counters, cudaStream_t s);
  FrameIo frame_io(const float* c_obs, const float* c_next) const {
    FrameIo f = io;
    f.c_obs = c_obs; f.c_next = c_next;
    return f;
  }
};

// The frame layout of BDQ's and DQN's replay: a plain fp32 row of E floats at a 16-byte stride (the gather's 128-bit loads
// stay aligned)
FrameIo plain_frames(int E);
// frame_capacity in [cap + 1, INT32_MAX] (frame indices are int32); `name` names it in the refusal
int check_frame_capacity(int64_t frame_cap, int64_t cap, const char* name);
// b2g_bdq_create2 / b2g_dqn_create2: replay NULL (the default layout) or check_frame_capacity, no 8-bit planes, one rank
int check_replay_cfg(const b2g_replay_cfg* replay, int64_t cap, int nranks);
// device bytes of a BDQ / DQN transition replay: the obs / next_obs rows or frames (and the frame indices), actions, rewards,
// dones
int64_t transition_replay_bytes(int64_t cap, int E, int A, int64_t frame_cap);
// a handle's fingerprint for its replay layout: one more field, replay_frames = frame_cap, with frames
std::vector<FpField> fp_with_frames(std::vector<FpField> fp, int64_t frame_cap);
// state_open_rms with the fingerprint of the handle's replay layout; a file of the other layout is refused with a message
// naming replay_frames
int state_open_replay(StateReader& rd, const char* path, uint32_t kind, const std::vector<FpField>& fp, int64_t frame_cap, bool owns_rms,
                      const char* rms_set_call);

}  // namespace b2g
