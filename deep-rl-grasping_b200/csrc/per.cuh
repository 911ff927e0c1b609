// Proportional prioritised replay on the device (per.cu), shared by the BDQ and DQN learners.
//
// [SB2] common/buffers.py PrioritizedReplayBuffer over common/segment_tree.py (Schaul et al. 2016), with the sum / min
// segment trees resident in HBM: leaves C..2C-1 (C = capacity rounded up to a power of two), node i = f(2i, 2i+1).  Sums are
// kept in float64 like the Python floats of the reference.
#pragma once
#include <cuda_runtime.h>

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

}  // namespace b2g
