// The flat transition replay of the BDQ and DQN learners, with proportional prioritised replay on the device (per.cu).
//
// [SB2] common/buffers.py PrioritizedReplayBuffer over common/segment_tree.py (Schaul et al. 2016), with the sum / min
// segment trees resident in HBM: leaves C..2C-1 (C = capacity rounded up to a power of two), node i = f(2i, 2i+1).  Sums are
// kept in float64 like the Python floats of the reference.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "state.cuh"

namespace b2g {

struct PerArgs {
  double* tsum; double* tmin; long long C;
  float* max_prio;                  // running max of the raw priorities (new transitions enter with it)
  const long long* counters;        // [4] rng step, [5] replay size
  unsigned long long seed;
  int B; float alpha, eps; const float* beta;
  int* indices; float* weights; float* prio_out;
  const float* td; int D;
};

// One CTA of round32(B) threads: draws B slots proportionally to priority (find_prefixsum_idx descent, Philox stream 2 at
// counters[4]) and their importance-sampling weights (p_i size)^-beta / max_w.  B <= 1024.
void per_sample_launch(const PerArgs& a, cudaStream_t s);
// One CTA of round32(n) threads (n <= 1024): writes n leaves and repairs their ancestors.  The leaves are slots[i], or
// (first_slot + i) % cap when slots == nullptr.  from_td != 0: raw priority sum_d |td[i * D + d]| + eps (also written to
// prio_out and folded into max_prio); else the running max_prio.  Leaf value raw^alpha.
void per_write_launch(const PerArgs& a, const int* slots, long long first_slot, long long cap, int n, int from_td, cudaStream_t s);
// Empty trees of n2 = 2C nodes (sum 0, min +inf) and max_prio = 1.
void per_init_launch(double* tsum, double* tmin, long long n2, float* max_prio, cudaStream_t s);

// Ring of cap transitions (obs [E], action [A], reward, done as float rows) and, with prioritised replay, its trees.  Row i of
// every ring is transition i; pos is the next row written, size the number of live rows.
struct TransitionReplay {
  float *obs = nullptr, *next = nullptr, *act = nullptr, *rew = nullptr, *done = nullptr;
  int64_t cap = 0, size = 0, pos = 0;
  int E = 0, A = 0;
  bool per = false;
  float alpha = 0.f, eps = 0.f;                         // priority exponent and the epsilon added to |TD|
  double *t_sum = nullptr, *t_min = nullptr;
  long long per_C = 0;
  float *max_prio = nullptr, *beta = nullptr, *prio_out = nullptr;   // prio_out: [B] priorities of the last sampled step

  // Allocates the rings, and the trees (empty, beta 0.4) when per; B is the batch of a sampled step.
  int init(std::vector<void*>& allocs, cudaStream_t s, int64_t cap, int E, int A, int B, bool per, float alpha, float eps);
  // The prioritised-replay arguments of a sampled step of B rows: draws into indices / weights, new priorities from td [B][D].
  PerArgs per_args(const long long* counters, unsigned long long seed, int B, int* indices, float* weights, const float* td, int D) const;
  // n transitions (host or device rows) at pos, in chunks that end at the ring's end; new rows enter at the running maximum
  // priority.  Then the size goes to counters[5] and the stream is drained.
  int add(const float* o, const float* a, const float* r, const float* nx, const float* d, int64_t n, long long* counters, cudaStream_t s);
  // Rows [first, first + n) (mod cap) enter at the running maximum priority ([SB2] PrioritizedReplayBuffer.add); nothing
  // without per.
  void insert_max_prio(int64_t first, int64_t n, cudaStream_t s) const;
  // pos and size after n more rows
  void advance(int64_t n);
  int set_beta(float beta, int device, cudaStream_t s);
  // b2g_*_get_last_per: slots of the last sampled step (uniform replay too), and with per its weights and new priorities
  int get_last(const int* indices, const float* weights, int B, int32_t* slots, float* w, float* p, int device, cudaStream_t s) const;
  // The training-state sections ROBS, RNXT, RACT, RREW, RDON, PERT, PERS of a replay holding `live` rows (rows [0, live) are the
  // live ones, the rings up to cap for the rest)
  std::vector<StateSection> state_sections(int64_t live) const;
  // size and pos a file may restore
  bool valid(int64_t size, int64_t pos) const { return size >= 0 && size <= cap && pos >= 0 && pos < cap && (size == cap || pos == size); }
};

}  // namespace b2g
