// Host bookkeeping of a replay whose transitions reference observation frames of a pool: the transition replay (per.cuh) of
// SAC, and of BDQ / DQN built with frames.  The frame rows themselves, and the kernels that check and write them, are
// FrameFmt / frame_check / frame_commit (common.cuh, replay.cu).
//
// Frames are allocated in FIFO order with monotone 64-bit ids; frame id f sits at f % frame_cap.  Transitions are numbered
// too: the live ones are [tail_seq, head_seq), transition t sits at slot t % cap.  When a new frame would overwrite one a live
// transition still references, the oldest transitions are dropped first (evicted counts them), so the live window can start
// mid-ring.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <deque>
#include <utility>
#include <vector>

namespace b2g {

struct FrameRing {
  int64_t frame_cap = 0;
  bool dedup = false;                // obs may share the previous call's next_obs frame (frame_cap < 2 cap)
  int64_t head_seq = 0, tail_seq = 0, next_fid = 0, evicted = 0;
  std::deque<std::pair<int64_t, int64_t>> lw;   // (transition, obs frame id): sliding-window minimum of the live obs frames
  std::vector<int64_t> prev_next;    // frame ids of the last call's next_obs rows

  // next frame id; a frame that would overwrite one a live transition references drops the oldest transitions first
  int64_t alloc_frame() {
    const int64_t f = next_fid++, over = f - frame_cap;
    while (head_seq > tail_seq) {
      while (lw.front().first < tail_seq) lw.pop_front();
      if (lw.front().second > over) break;
      ++tail_seq; ++evicted;
    }
    return f;
  }
  // One more transition in a ring of cap slots: its obs frame *of (the candidate frame cand >= 0 when sharing is on and it
  // outlives the allocation of this transition's next_obs frame, else a new one) and its next_obs frame *nf.  Returns whether
  // the obs frame is shared.
  bool add_transition(int64_t cap, int64_t cand, int64_t* of, int64_t* nf) {
    if (head_seq - tail_seq == cap) ++tail_seq;                       // the ring's own replacement
    const bool share = dedup && cand >= 0 && cand >= next_fid + 1 - frame_cap;
    *of = share ? cand : alloc_frame();
    *nf = alloc_frame();
    while (!lw.empty() && lw.back().second >= *of) lw.pop_back();
    lw.emplace_back(head_seq++, *of);
    return share;
  }
  int64_t size() const { return head_seq - tail_seq; }
  // frames from the oldest one a live transition references to the newest
  int64_t live_frames() const {
    if (size() <= 0) return 0;
    int64_t lo = next_fid;
    for (const auto& q : lw) if (q.first >= tail_seq) { lo = q.second; break; }
    return next_fid - lo;
  }
  // oldest frame a training-state file must hold: the oldest one a live transition references, or a previous next_obs frame
  // the next call may still share
  int64_t frame_lo() const {
    int64_t lo = next_fid - live_frames();
    for (int64_t p : prev_next) if (p > next_fid - frame_cap) lo = std::min(lo, p);
    return lo;
  }
  // as stored in a training-state file: size, head_seq, tail_seq, next_fid, evicted, |lw|, |prev_next|, lw pairs, prev_next
  std::vector<int64_t> pack() const {
    std::vector<int64_t> v = {size(), head_seq, tail_seq, next_fid, evicted, (int64_t)lw.size(), (int64_t)prev_next.size()};
    for (const auto& q : lw) { v.push_back(q.first); v.push_back(q.second); }
    v.insert(v.end(), prev_next.begin(), prev_next.end());
    return v;
  }
  // the inverse of pack() into this ring (frame_cap and dedup kept); false when v is not a consistent bookkeeping of a ring
  // of cap slots
  bool unpack(const int64_t* v, size_t n, int64_t cap) {
    if (n < 7) return false;
    const int64_t n_lw = v[5], n_prev = v[6];
    if (n_lw < 0 || n_prev < 0 || (int64_t)n != 7 + 2 * n_lw + n_prev || v[0] != v[1] - v[2] || v[0] < 0 || v[0] > cap || v[2] < 0 ||
        v[3] < 0 || v[4] < 0)
      return false;
    head_seq = v[1]; tail_seq = v[2]; next_fid = v[3]; evicted = v[4];
    lw.clear();
    for (int64_t i = 0; i < n_lw; ++i) lw.emplace_back(v[7 + 2 * i], v[8 + 2 * i]);
    prev_next.assign(v + 7 + 2 * n_lw, v + n);
    const int64_t lo = frame_lo();
    return lo >= 0 && lo <= next_fid && next_fid - lo <= frame_cap;
  }
};

}  // namespace b2g
