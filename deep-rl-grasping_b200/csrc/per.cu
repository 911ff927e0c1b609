// Prioritised-replay kernels and the transition replay (declarations and the tree layout in per.cuh).
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "host.cuh"
#include "per.cuh"

namespace b2g {
namespace {

// one CTA, B threads: draws B slots proportionally to priority (find_prefixsum_idx descent) and their IS weights
__global__ void per_sample_kernel(PerArgs a) {
  const int b = threadIdx.x;
  if (b >= a.B) return;
  const unsigned long long step = (unsigned long long)a.counters[4];
  const long long size = a.counters[5];
  const uint4 r = philox4x32_10(make_uint4((unsigned)step, (unsigned)(step >> 32), (unsigned)(b >> 2), 2u), make_uint2((unsigned)a.seed, (unsigned)(a.seed >> 32)));
  const unsigned v = (b & 3) == 0 ? r.x : (b & 3) == 1 ? r.y : (b & 3) == 2 ? r.z : r.w;
  const double total = a.tsum[1];
  double mass = ((double)v + 0.5) * (1.0 / 4294967296.0) * total;
  long long node = 1;
  while (node < a.C) {
    const double left = a.tsum[2 * node];
    if (left > mass) node = 2 * node;
    else { mass -= left; node = 2 * node + 1; }
  }
  long long idx = node - a.C;
  if (a.ring_cap > 0) {                                  // live window [counters[6], + size) mod ring_cap; other leaves are 0
    if (a.tsum[a.C + idx] == 0.0) idx = ring_slot(a.counters[6], (int)(size - 1), a.ring_cap);
  } else if (idx >= size) idx = size - 1;                // (rounding at the right edge of the occupied range)
  const double beta = (double)a.beta[0];
  const double p_min = a.tmin[1] / total;
  const double max_w = pow(p_min * (double)size, -beta);
  const double p = a.tsum[a.C + idx] / total;
  a.indices[b] = (int)idx;
  a.weights[b] = (float)(pow(p * (double)size, -beta) / max_w);
}

// one CTA: writes `n` leaves and repairs their ancestors level by level (siblings recomputed redundantly: same values)
__global__ void per_write_kernel(PerArgs a, const int* __restrict__ slots, long long first_slot, long long cap, int n, int from_td) {
  const int i = threadIdx.x;
  long long leaf = 0;
  if (i < n) {
    const long long slot = slots ? (long long)slots[i] : (first_slot + i) % cap;
    float raw = 0.f;
    if (from_td == 2) {                                   // the slot left the replay: out of both trees
      leaf = a.C + slot;
      a.tsum[leaf] = 0.0; a.tmin[leaf] = INFINITY;
    } else if (from_td) {
      float s = 0.f;
      for (int d = 0; d < a.D; ++d) s += fabsf(a.td[i * a.D + d]);
      raw = s + a.eps;
      atomicMax(reinterpret_cast<int*>(a.max_prio), __float_as_int(raw));      // positive floats order like their bit patterns
      if (a.prio_out) a.prio_out[i] = raw;
    } else raw = a.max_prio[0];
    if (from_td != 2) {
      const double pr = pow((double)raw, (double)a.alpha);
      leaf = a.C + slot;
      a.tsum[leaf] = pr; a.tmin[leaf] = pr;
    }
  }
  __syncthreads();
  for (long long span = a.C; span > 1; span >>= 1) {
    if (i < n) {
      leaf >>= 1;
      a.tsum[leaf] = a.tsum[2 * leaf] + a.tsum[2 * leaf + 1];
      a.tmin[leaf] = fmin(a.tmin[2 * leaf], a.tmin[2 * leaf + 1]);
    }
    __syncthreads();
  }
}

__global__ void per_init_kernel(double* tsum, double* tmin, long long n2, float* max_prio) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n2; i += (long long)gridDim.x * blockDim.x) { tsum[i] = 0.0; tmin[i] = INFINITY; }
  if (blockIdx.x == 0 && threadIdx.x == 0) max_prio[0] = 1.0f;
}

}  // namespace

void per_sample_launch(const PerArgs& a, cudaStream_t s) { per_sample_kernel<<<1, ((a.B + 31) / 32) * 32, 0, s>>>(a); }

void per_write_launch(const PerArgs& a, const int* slots, long long first_slot, long long cap, int n, int from_td, cudaStream_t s) {
  per_write_kernel<<<1, ((n + 31) / 32) * 32, 0, s>>>(a, slots, first_slot, cap, n, from_td);
}

void per_init_launch(double* tsum, double* tmin, long long n2, float* max_prio, cudaStream_t s) {
  per_init_kernel<<<256, 256, 0, s>>>(tsum, tmin, n2, max_prio);
}

FrameIo plain_frames(int E) {
  FrameIo f{};
  f.npx = 0; f.Ci = 1; f.Ec = E;         // fmt {}: the whole row is the fp32 tail
  f.frame_bytes = ((int64_t)E * (int64_t)sizeof(float) + 15) / 16 * 16;
  return f;
}

int TransitionReplay::init(std::vector<void*>& allocs, cudaStream_t s, int64_t cap_, int E_, int A_, int B, bool per_, float alpha_,
                           float eps_, int64_t frame_cap, const FrameIo& layout, int stage_rows_) {
  cap = cap_; E = E_; A = A_; per = per_; alpha = alpha_; eps = eps_;
  if (cudaMallocHost((void**)&h_rc, 2 * sizeof(long long)) != cudaSuccess) return b2g_fail(B2G_ECUDA, "replay staging");
  if (frame_cap > 0) {
    ring.frame_cap = frame_cap;
    ring.dedup = frame_cap < 2 * cap;     // at 2 cap every transition has two frames of its own: sharing would save nothing
    io = layout;
    // one commit launch writes distinct transition slots and distinct frames
    stage_rows = (int)std::min<int64_t>({(int64_t)stage_rows_, cap, frame_cap / 2});
    if (int rc = dev_alloc(allocs, s, &io.frames, (size_t)(frame_cap * io.frame_bytes))) return rc;
    if (int rc = dev_alloc(allocs, s, &r_ofr, cap)) return rc;
    if (int rc = dev_alloc(allocs, s, &r_nfr, cap)) return rc;
    if (int rc = dev_alloc(allocs, s, &c_obs, (size_t)stage_rows * io.Ec)) return rc;
    if (int rc = dev_alloc(allocs, s, &c_next, (size_t)stage_rows * io.Ec)) return rc;
    if (int rc = dev_alloc(allocs, s, &d_plan, 4 * (size_t)stage_rows)) return rc;
    if (cudaMallocHost((void**)&h_plan, 4 * (size_t)stage_rows * sizeof(int)) != cudaSuccess) return b2g_fail(B2G_ECUDA, "replay staging");
  } else {
    if (int rc = dev_alloc(allocs, s, &obs, cap * E)) return rc;
    if (int rc = dev_alloc(allocs, s, &next, cap * E)) return rc;
  }
  if (int rc = dev_alloc(allocs, s, &act, cap * A)) return rc;
  if (int rc = dev_alloc(allocs, s, &rew, cap)) return rc;
  if (int rc = dev_alloc(allocs, s, &done, cap)) return rc;
  if (int rc = dev_alloc(allocs, s, &beta, 1)) return rc;
  if (int rc = dev_alloc(allocs, s, &max_prio, 1)) return rc;
  if (int rc = dev_alloc(allocs, s, &prio_out, B)) return rc;
  if (!per) return 0;
  per_C = 1;
  while (per_C < cap) per_C <<= 1;
  if (int rc = dev_alloc(allocs, s, &t_sum, 2 * per_C)) return rc;
  if (int rc = dev_alloc(allocs, s, &t_min, 2 * per_C)) return rc;
  per_init_launch(t_sum, t_min, 2 * per_C, max_prio, s);
  const float beta0 = 0.4f;
  CK(cudaMemcpyAsync(beta, &beta0, sizeof(float), cudaMemcpyHostToDevice, s));
  return 0;
}

void TransitionReplay::release() {
  if (h_plan) cudaFreeHost(h_plan);
  if (h_rc) cudaFreeHost(h_rc);
  h_plan = nullptr; h_rc = nullptr;
}

PerArgs TransitionReplay::per_args(const long long* counters, unsigned long long seed, int B, int* indices, float* weights, const float* td,
                                   int D) const {
  PerArgs pr{};
  pr.tsum = t_sum; pr.tmin = t_min; pr.C = per_C; pr.max_prio = max_prio; pr.counters = counters; pr.seed = seed;
  pr.B = B; pr.alpha = alpha; pr.eps = eps; pr.beta = beta; pr.indices = indices; pr.weights = weights;
  pr.prio_out = prio_out; pr.td = td; pr.D = D; pr.ring_cap = ring_cap();
  return pr;
}

void TransitionReplay::insert_max_prio(int64_t first, int64_t n, cudaStream_t s) const {
  if (!per) return;
  const PerArgs pr = per_args(nullptr, 0, 0, nullptr, nullptr, nullptr, 0);
  for (int64_t o = 0; o < n; o += 1024) per_write_launch(pr, nullptr, first + o, cap, (int)std::min<int64_t>(1024, n - o), 0, s);
}

void TransitionReplay::advance(int64_t n) {
  pos = (pos + n) % cap;
  size = std::min(cap, size + n);
}

void TransitionReplay::gather_args(GatherArgs& g, bool with_next) const {
  g.act = with_next ? act : nullptr; g.rew = rew; g.done = done;
  if (!framed()) {
    g.obs = obs; g.next_obs = with_next ? next : nullptr;
    return;
  }
  g.obs = nullptr; g.next_obs = nullptr;
  g.frames = io.frames; g.frame_bytes = io.frame_bytes; g.obs_frame = r_ofr; g.next_frame = with_next ? r_nfr : nullptr;
  g.fmt = io.fmt; g.ring_cap = cap;
}

int TransitionReplay::commit(const float* co, const float* cn, int m, const int64_t* cand, const float* a, const float* r, const float* d,
                             int64_t* next_ids, cudaStream_t s) {
  const int64_t FC = ring.frame_cap, first = ring.head_seq, fid0 = ring.next_fid, tail0 = ring.tail_seq;
  for (int i = 0; i < m; ++i) {
    int64_t of, nf;
    const bool share = ring.add_transition(cap, cand[i], &of, &nf);
    h_plan[i] = (int)(of % FC); h_plan[m + i] = share ? 0 : 1; h_plan[2 * m + i] = (int)(nf % FC);
    next_ids[i] = nf;
  }
  if (ring.dedup) CK(cudaMemcpyAsync(d_plan, h_plan, 3 * m * sizeof(int), cudaMemcpyHostToDevice, s));
  frame_commit_launch(frame_io(co, cn), ring.dedup ? d_plan : nullptr, fid0, FC, m, r_ofr, r_nfr, first, cap, s);
  for (int64_t k = 0; k < m;) {          // act / rew / done into slots (first + k) % cap, in at most two pieces
    const int64_t p = (first + k) % cap, len = std::min<int64_t>(m - k, cap - p);
    CK(cudaMemcpyAsync(act + p * A, a + k * A, len * A * sizeof(float), cudaMemcpyDefault, s));
    CK(cudaMemcpyAsync(rew + p, r + k, len * sizeof(float), cudaMemcpyDefault, s));
    CK(cudaMemcpyAsync(done + p, d + k, len * sizeof(float), cudaMemcpyDefault, s));
    k += len;
  }
  insert_max_prio(first % cap, m, s);
  if (per) {      // transitions dropped early, whose slots no row of this chunk took over, leave the trees (after the insert)
    const int64_t lo = std::max(tail0, ring.head_seq - cap), hi = ring.tail_seq;
    const PerArgs pr = per_args(nullptr, 0, 0, nullptr, nullptr, nullptr, 0);
    for (int64_t o = lo; o < hi; o += 1024) per_write_launch(pr, nullptr, o % cap, cap, (int)std::min<int64_t>(1024, hi - o), 2, s);
  }
  return 0;
}

int TransitionReplay::finish(std::vector<int64_t>& next_ids, long long* counters, cudaStream_t s) {
  ring.prev_next.swap(next_ids);
  size = ring.size();
  pos = ring.head_seq % cap;
  h_rc[0] = size;
  h_rc[1] = size == cap ? 0 : ring.tail_seq % cap;     // the first live slot
  CK(cudaMemcpyAsync(counters + 5, h_rc, 2 * sizeof(long long), cudaMemcpyHostToDevice, s));
  return 0;
}

int TransitionReplay::add_linked(const float* co, const float* cn, const int64_t* cand, const float* a, const float* r, const float* d, int n,
                                 int64_t* next_fid, long long* counters, cudaStream_t s) {
  std::vector<int64_t> next_ids((size_t)n);
  for (int64_t c0 = 0; c0 < n; c0 += stage_rows) {
    const int m = (int)std::min<int64_t>(stage_rows, n - c0);
    if (c0 > 0) CK(cudaStreamSynchronize(s));        // the previous chunk's plan upload has left h_plan
    if (int rc = commit(co + c0 * io.Ec, cn + c0 * io.Ec, m, cand + c0, a + c0 * A, r + c0, d + c0, next_ids.data() + c0, s)) return rc;
  }
  std::copy(next_ids.begin(), next_ids.end(), next_fid);
  return finish(next_ids, counters, s);
}

int TransitionReplay::add(const float* o, const float* a, const float* r, const float* nx, const float* d, int64_t n, long long* counters,
                          cudaStream_t s, const RowLoader& load) {
  if (framed()) {
    const int64_t R = stage_rows, FC = ring.frame_cap;
    if (ring.dedup && 2 * n > FC) return b2g_fail(B2G_EINVAL, std::string("replay_add: 2 n rows exceed ") + frames_name);
    const bool u8 = io.fmt.n8 > 0;
    const FrameIo fio = frame_io(c_obs, c_next);
    int* flags = h_plan + 3 * R;
    // rows [c0, c0 + m) -> the compact staging, then (when sharing frames or checking 8-bit values) frame_check -> flags,
    // synchronised
    auto stage = [&](int64_t c0, int m, bool check) -> int {
      if (c0 > 0) CK(cudaStreamSynchronize(s));        // the previous chunk's plan upload has left h_plan
      for (int w = 0; w < 2; ++w) {
        const float* src = (w ? nx : o) + c0 * E;
        float* dst = w ? c_next : c_obs;
        if (load) {
          if (int rc = load(src, dst, m)) return rc;
        } else CK(cudaMemcpyAsync(dst, src, m * io.Ec * sizeof(float), cudaMemcpyDefault, s));
      }
      if (!check) return 0;
      for (int i = 0; i < m; ++i) {      // candidate frame of row i: the previous call's next_obs of row i, while it still exists
        const int64_t p = c0 + i < (int64_t)ring.prev_next.size() ? ring.prev_next[c0 + i] : -1;
        h_plan[i] = ring.dedup && p >= 0 && p > ring.next_fid - FC ? (int)(p % FC) : -1;
      }
      CK(cudaMemcpyAsync(d_plan, h_plan, m * sizeof(int), cudaMemcpyHostToDevice, s));
      frame_check_launch(fio, d_plan, d_plan + 3 * R, m, s);
      CK(cudaMemcpyAsync(flags, d_plan + 3 * R, m * sizeof(int), cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      for (int i = 0; i < m; ++i)
        if (flags[i] & 2) return b2g_fail(B2G_EINVAL, "replay_add: a value of an 8-bit plane is not an integer in [0, 255]");
      return 0;
    };
    // a call larger than the staging validates every row before it stores the first one
    if (u8 && n > R)
      for (int64_t c0 = 0; c0 < n; c0 += R)
        if (int rc = stage(c0, (int)std::min<int64_t>(R, n - c0), true)) return rc;
    std::vector<int64_t> next_ids((size_t)n), cand((size_t)R);
    for (int64_t c0 = 0; c0 < n; c0 += R) {
      const int m = (int)std::min<int64_t>(R, n - c0);
      if (int rc = stage(c0, m, ring.dedup || (u8 && n <= R))) return rc;
      for (int i = 0; i < m; ++i)        // the previous call's next_obs of row i, where frame_check found it equal bit for bit
        cand[i] = ring.dedup && (flags[i] & 1) ? ring.prev_next[c0 + i] : -1;
      if (int rc = commit(c_obs, c_next, m, cand.data(), a + c0 * A, r + c0, d + c0, next_ids.data() + c0, s)) return rc;
    }
    if (int rc = finish(next_ids, counters, s)) return rc;
    CK(cudaStreamSynchronize(s));
    return 0;
  }
  for (int64_t done_n = 0; done_n < n;) {
    const int64_t chunk = std::min(n - done_n, cap - pos);
    CK(cudaMemcpyAsync(obs + pos * E, o + done_n * E, chunk * E * sizeof(float), cudaMemcpyDefault, s));
    CK(cudaMemcpyAsync(next + pos * E, nx + done_n * E, chunk * E * sizeof(float), cudaMemcpyDefault, s));
    CK(cudaMemcpyAsync(act + pos * A, a + done_n * A, chunk * A * sizeof(float), cudaMemcpyDefault, s));
    CK(cudaMemcpyAsync(rew + pos, r + done_n, chunk * sizeof(float), cudaMemcpyDefault, s));
    CK(cudaMemcpyAsync(done + pos, d + done_n, chunk * sizeof(float), cudaMemcpyDefault, s));
    insert_max_prio(pos, chunk, s);
    advance(chunk);
    done_n += chunk;
  }
  h_rc[0] = size;
  CK(cudaMemcpyAsync(counters + 5, h_rc, sizeof(long long), cudaMemcpyHostToDevice, s));
  CK(cudaStreamSynchronize(s));
  return 0;
}

int TransitionReplay::set_beta(float b, int device, cudaStream_t s) {
  CK(cudaSetDevice(device));
  CK(cudaStreamSynchronize(s));
  CK(cudaMemcpy(beta, &b, sizeof(float), cudaMemcpyHostToDevice));
  return 0;
}

int TransitionReplay::get_last(const int* indices, const float* weights, int B, int32_t* slots, float* w, float* p, int device,
                               cudaStream_t s) const {
  CK(cudaSetDevice(device));
  CK(cudaStreamSynchronize(s));
  if (slots) CK(cudaMemcpy(slots, indices, B * sizeof(int32_t), cudaMemcpyDeviceToHost));
  if (w) CK(cudaMemcpy(w, weights, B * sizeof(float), cudaMemcpyDeviceToHost));
  if (p) CK(cudaMemcpy(p, prio_out, B * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

int TransitionReplay::get(int64_t slot, float* o, float* a, float* r, float* nx, float* d, int32_t* frame_ids, int device,
                          cudaStream_t s) const {
  const int64_t first = framed() && size < cap ? ring.tail_seq % cap : 0;
  if (slot < 0 || slot >= cap || ((slot - first) % cap + cap) % cap >= size) return b2g_fail(B2G_EINVAL, "replay slot is not live");
  CK(cudaSetDevice(device));
  CK(cudaStreamSynchronize(s));
  int fr[2] = {-1, -1};
  if (framed()) {
    CK(cudaMemcpy(&fr[0], r_ofr + slot, sizeof(int), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(&fr[1], r_nfr + slot, sizeof(int), cudaMemcpyDeviceToHost));
  }
  std::vector<float> frame(framed() ? io.frame_bytes / sizeof(float) : 0);    // frame strides are whole floats
  for (int w = 0; w < 2; ++w) {
    float* dst = w ? nx : o;
    if (!dst) continue;
    if (!framed()) {
      CK(cudaMemcpy(dst, (w ? next : obs) + slot * E, E * sizeof(float), cudaMemcpyDeviceToHost));
      continue;
    }
    CK(cudaMemcpy(frame.data(), io.frames + (size_t)fr[w] * io.frame_bytes, io.frame_bytes, cudaMemcpyDeviceToHost));
    const unsigned char* f = reinterpret_cast<const unsigned char*>(frame.data());
    for (int e = 0; e < io.Ec; ++e) dst[e] = frame_elem(f, io.fmt, io.npx, io.Ci, e);
  }
  if (a) CK(cudaMemcpy(a, act + slot * A, A * sizeof(float), cudaMemcpyDeviceToHost));
  if (r) CK(cudaMemcpy(r, rew + slot, sizeof(float), cudaMemcpyDeviceToHost));
  if (d) CK(cudaMemcpy(d, done + slot, sizeof(float), cudaMemcpyDeviceToHost));
  if (frame_ids) { frame_ids[0] = fr[0]; frame_ids[1] = fr[1]; }
  return 0;
}

void TransitionReplay::info(int64_t* capacity, int64_t* sz, int64_t* frame_capacity, int64_t* live_frames, int64_t* bytes,
                            int64_t* evicted_early) const {
  if (capacity) *capacity = cap;
  if (sz) *sz = size;
  if (frame_capacity) *frame_capacity = ring.frame_cap;
  if (live_frames) *live_frames = ring.live_frames();
  if (bytes) {
    const int64_t fb = sizeof(float);
    *bytes = (framed() ? ring.frame_cap * io.frame_bytes + 2 * cap * (int64_t)sizeof(int) : 2 * cap * E * fb) + cap * (A + 2) * fb;
  }
  if (evicted_early) *evicted_early = ring.evicted;
}

int check_frame_capacity(int64_t frame_cap, int64_t cap, const char* name) {
  if (frame_cap < cap + 1) return b2g_fail(B2G_EINVAL, std::string(name) + " must be at least buffer_capacity + 1");
  if (frame_cap > INT32_MAX) return b2g_fail(B2G_EINVAL, std::string(name) + " must fit in int32 (frame indices)");
  return 0;
}

int check_replay_cfg(const b2g_replay_cfg* r, int64_t cap, int nranks) {
  if (!r) return 0;
  if (int rc = check_frame_capacity(r->frame_capacity, cap, "frame_capacity (replay_frames)")) return rc;
  if (r->u8_plane_mask)
    return b2g_fail(B2G_EINVAL, "u8_plane_mask: the BDQ / DQN replay stores fp32 observation vectors (8-bit planes are SAC's CNN rows)");
  if (nranks > 1) return b2g_fail(B2G_EINVAL, "replay frames (replay_frames) are not built for data-parallel learners (nranks > 1)");
  return 0;
}

int64_t transition_replay_bytes(int64_t cap, int E, int A, int64_t frame_cap) {
  const int64_t fb = sizeof(float);
  const int64_t rows = frame_cap > 0 ? frame_cap * plain_frames(E).frame_bytes + 2 * cap * (int64_t)sizeof(int) : 2 * cap * E * fb;
  return rows + cap * (A + 2) * fb;
}

std::vector<FpField> fp_with_frames(std::vector<FpField> fp, int64_t frame_cap) {
  if (frame_cap > 0) fp.push_back(fp_int("replay_frames", frame_cap));
  return fp;
}

int state_open_replay(StateReader& rd, const char* path, uint32_t kind, const std::vector<FpField>& fp, int64_t frame_cap, bool owns_rms,
                      const char* rms_set_call) {
  const int rc = state_open_rms(rd, path, kind, fp_with_frames(fp, frame_cap), owns_rms, rms_set_call);
  if (rc == 0) return 0;
  const std::string msg = g_b2g_err;
  const int has = state_fp_field(path, kind, "replay_frames");
  if (has == 1 && frame_cap == 0)
    return b2g_fail(B2G_EINVAL, "the state file holds a replay of frames (replay_frames); this handle was created without them");
  if (has == 0 && frame_cap > 0)
    return b2g_fail(B2G_EINVAL, "the state file holds the default replay layout; this handle keeps its replay in " + std::to_string(frame_cap) +
                                    " frames (replay_frames)");
  return b2g_fail(rc, msg);
}

std::vector<int64_t> TransitionReplay::state_host(int64_t n_updates, int64_t eps_bits) const {
  std::vector<int64_t> hv = {size, pos, n_updates, eps_bits};
  if (framed()) for (int64_t v : ring.pack()) hv.push_back(v);
  return hv;
}

int TransitionReplay::state_host_read(StateReader& rd, std::vector<int64_t>* hv, FrameRing* rg) const {
  const uint64_t hb = rd.bytes(0);
  if (framed() ? hb % 8 || hb < 11 * 8 || hb > (uint64_t)(11 + 2 * cap + 4 * ring.frame_cap) * 8 : hb != 4 * 8)
    return b2g_fail(B2G_EINVAL, "training-state section lengths do not match this handle's configuration");
  hv->resize(hb / 8);
  if (int rc = rd.read_host(0, hv->data(), hb)) return rc;
  const int64_t* v = hv->data();
  *rg = ring;
  const bool ok = framed() ? rg->unpack(v + 4, hv->size() - 4, cap) && v[0] == rg->size() && v[1] == rg->head_seq % cap : valid(v[0], v[1]);
  if (!ok || v[2] < 0) return b2g_fail(B2G_EINVAL, "corrupt replay bookkeeping in the training-state file");
  return 0;
}

std::vector<StateSection> TransitionReplay::state_sections(int64_t live, int64_t lo, int64_t hi) const {
  const size_t fb = sizeof(float);
  if (framed()) {
    std::vector<StateSection> s(6);
    s[0].tag = state_tag("ROFR"); s[0].pieces = {dev_piece(r_ofr, cap * sizeof(int))};
    s[1].tag = state_tag("RNFR"); s[1].pieces = {dev_piece(r_nfr, cap * sizeof(int))};
    s[2].tag = state_tag("RACT"); s[2].pieces = {dev_piece(act, cap * A * fb)};
    s[3].tag = state_tag("RREW"); s[3].pieces = {dev_piece(rew, cap * fb)};
    s[4].tag = state_tag("RDON"); s[4].pieces = {dev_piece(done, cap * fb)};
    s[5].tag = state_tag("FRMS");
    for (int64_t f = lo; f < hi;) {      // frames [lo, hi): at most two contiguous ranges, each stored at id % frame_cap
      const int64_t p = f % ring.frame_cap, n = std::min(hi - f, ring.frame_cap - p);
      s[5].pieces.push_back(dev_piece(io.frames + p * io.frame_bytes, (size_t)(n * io.frame_bytes)));
      f += n;
    }
    return s;
  }
  (void)lo; (void)hi;
  std::vector<StateSection> s(5);
  s[0].tag = state_tag("ROBS"); s[0].pieces = {dev_piece(obs, live * E * fb)};
  s[1].tag = state_tag("RNXT"); s[1].pieces = {dev_piece(next, live * E * fb)};
  s[2].tag = state_tag("RACT"); s[2].pieces = {dev_piece(act, cap * A * fb)};
  s[3].tag = state_tag("RREW"); s[3].pieces = {dev_piece(rew, cap * fb)};
  s[4].tag = state_tag("RDON"); s[4].pieces = {dev_piece(done, cap * fb)};
  return s;
}

std::vector<StateSection> TransitionReplay::per_sections() const {
  std::vector<StateSection> s(2);
  s[0].tag = state_tag("PERT");
  if (per) s[0].pieces = {dev_piece(t_sum, 2 * per_C * sizeof(double)), dev_piece(t_min, 2 * per_C * sizeof(double))};
  s[1].tag = state_tag("PERS"); s[1].pieces = {dev_piece(max_prio, sizeof(float)), dev_piece(beta, sizeof(float))};
  return s;
}

}  // namespace b2g

extern "C" int64_t b2g_transition_replay_bytes(int64_t buffer_capacity, int obs_dim, int act_width, int64_t frame_capacity) {
  return b2g::transition_replay_bytes(buffer_capacity, obs_dim, act_width, frame_capacity);
}
