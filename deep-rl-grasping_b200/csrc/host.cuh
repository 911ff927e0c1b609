// Host runtime shared by the learner and encoder handles (host.cu): error state, device check, tracked device allocations,
// offset tables, gather-GEMM descriptor groups, CUDA-graph capture, learning-rate upload, the named-parameter table of the BDQ,
// DQN, PPO2 and TRPO handles and NCCL through dlopen.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <functional>
#include <map>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/b200grasp.h"
#include "common.cuh"

// Text behind b2g_last_error(): b2g_fail sets it and returns `code`.
extern thread_local std::string g_b2g_err;
int b2g_fail(int code, const std::string& msg);
// Returns B2G_ECUDA from the enclosing function when a CUDA runtime call fails.
#define CK(call)                                                                                  \
  do {                                                                                            \
    cudaError_t e_ = (call);                                                                      \
    if (e_ != cudaSuccess)                                                                        \
      return b2g_fail(B2G_ECUDA, std::string(#call) + ": " + cudaGetErrorString(e_) + " @" + __FILE__ + ":" + \
                                     std::to_string(__LINE__));                                   \
  } while (0)

// Returns B2G_ESTATE from the enclosing entry point when a failed training-state load left handle h unusable.
#define B2G_USABLE(h)                                                                                        \
  do {                                                                                                       \
    if ((h) && (h)->broken)                                                                                  \
      return b2g_fail(B2G_ESTATE, "handle unusable: a training-state load failed part way (load a state again or destroy it)"); \
  } while (0)

namespace b2g {

// The device exists, is made current and is a Hopper part (sm_90); *num_sms receives its SM count when asked for.
int check_device(int device, int* num_sms = nullptr);

// `count` elements of T (at least one) on the device, zeroed on stream s unless zero == false.  The pointer joins `allocs`,
// which the owning handle frees on destroy.
template <class T>
int dev_alloc(std::vector<void*>& allocs, cudaStream_t s, T** ptr, size_t count, bool zero = true) {
  void* q = nullptr;
  CK(cudaMalloc(&q, std::max<size_t>(count, 1) * sizeof(T)));
  allocs.push_back(q);
  if (zero) CK(cudaMemsetAsync(q, 0, std::max<size_t>(count, 1) * sizeof(T), s));
  *ptr = (T*)q;
  return 0;
}

// Offset table -> device, synchronously (v may be a temporary).  host_copy, when given, keeps v under the device pointer.
int upload_table(std::vector<void*>& allocs, cudaStream_t s, const std::vector<int>& v, const int** out,
                 std::map<const int*, std::vector<int>>* host_copy = nullptr);
std::vector<int> iota_tab(int n, int stride = 1, int base = 0);     // base + i * stride

// C[cM[m] + cN[n]] = sum_r A[aM[m] + aR[r]] * B[bR[r] + bN[n]] with the given flags; every optional operand unset, alpha = 1
GemmDesc gemm_desc(const float* A, const int* aM, const int* aR, const float* B, const int* bR, const int* bN, float* C,
                   const int* cM, const int* cN, int M, int N, int R, int flags, int splitR = 1);
// Tile grid of every descriptor of a grouped launch (bm x bn output tiles, splitR slices each), their tile_start / tile_count
// and the group's total_tiles; then the descriptors are copied to g.dev (allocated on the first call), synchronously.
int finalize_tiles(GemmGroup& g, std::vector<void*>& allocs, cudaStream_t s, int bm = GG_SIMT_BM, int bn = GG_SIMT_BN);

// Identity of the column tables of a wgmma-engine descriptor, (cN, kN, bias under GG_EPI_BIAS_RELU, N) -> id: equal ids share the
// column tables the gg_tc.cu epilogue stages, so consecutive tiles of such descriptors do not re-stage them.
using ColIds = std::map<std::tuple<const void*, const void*, const void*, int>, int>;
// The descriptor fields derived from its tables rather than given by the caller: GG_CN_AFFINE4 (set when the host copies in
// host_tabs show N % 4 == 0, cN contiguous in aligned groups of 4 and cM a multiple of 4, and under GG_EPI_MASK or
// GG_EPI_LRELU_GRAD the same of kN and kM when given) and col_id (new tables take the next id of col_ids).
void gg_tc_columns(GemmDesc& d, const std::map<const int*, std::vector<int>>& host_tabs, ColIds& col_ids);

// Captures what issue() enqueues on s into a graph and instantiates it into *exec.  A failing issue() ends the capture and
// returns its code.
int capture_graph(cudaStream_t s, const std::function<int()>& issue, cudaGraphExec_t* exec);

// Learning rate -> the device scalar the prep kernel reads; only when it changed (the stream is drained first).
int upload_lr(float* d_lr, float* cur_lr, float lr, cudaStream_t s);

// ---- named parameters of the BDQ, DQN, PPO2 and TRPO handles: the variables of the zip, in its order, and where each one lives
struct ParamEntry {
  std::string name;            // full zip name
  int64_t rows, cols;          // zip shape [rows, cols]; rows = 1 for ndim 1, rows = cols = 1 for a scalar
  int ndim;
  int stride;                  // device row stride (floats)
  int64_t off;                 // float offset into the parameter arena, and into the gradient arena when grad
  bool grad;                   // the gradient arena holds this variable
  float* scalar;               // a host scalar (bdq/eps, deepq/eps) instead of arena rows
};
enum class ParamCopy { Get, Set, GetGrad };

class ParamTable {
 public:
  void add(const std::string& name, int64_t rows, int64_t cols, int ndim, int stride, int64_t off, bool grad);
  void add_scalar(const std::string& name, float* v);
  // copies of entries [first, first + n) renamed from_scope... -> to_scope..., at off + shift, without gradient (target nets)
  void add_copies(int first, int n, const std::string& from_scope, const std::string& to_scope, int64_t shift);
  int count() const { return (int)entries_.size(); }
  const std::vector<ParamEntry>& entries() const { return entries_; }
  int64_t off(const std::string& name) const { return entries_[index_.at(name)].off; }
  // b2g_*_param_info
  int info(int idx, char* name, size_t name_cap, int64_t* rows, int64_t* cols, int32_t* ndim) const;
  // b2g_*_get_param / _set_param / _get_grad: a trailing ":0" is ignored; the stream is drained, then the rows are repacked
  // between the zip layout and the device row stride
  int copy(const char* name, ParamCopy mode, float* P, float* G, float* host, size_t numel, int device, cudaStream_t s) const;

 private:
  std::vector<ParamEntry> entries_;
  std::map<std::string, int> index_;
};

// The next 32-float-aligned arena range of n floats: returns its offset and advances off.
inline int64_t arena_take(int64_t& off, int64_t n) { const int64_t o = off; off += (n + 31) / 32 * 32; return o; }

// The parameter ABI of handle h (members params, P, G, cfg.device, stream, broken).
template <class H>
int param_count(const H* h) { B2G_USABLE(h); return h ? h->params.count() : 0; }
template <class H>
int param_info(const H* h, int idx, char* name, size_t name_cap, int64_t* rows, int64_t* cols, int32_t* ndim) {
  B2G_USABLE(h);
  return h ? h->params.info(idx, name, name_cap, rows, cols, ndim) : b2g_fail(B2G_EINVAL, "bad tensor index");
}
template <class H>
int param_copy(H* h, const char* name, ParamCopy mode, float* host, size_t numel) {
  B2G_USABLE(h);
  if (!h) return b2g_fail(B2G_EINVAL, "NULL argument");
  return h->params.copy(name, mode, h->P, h->G, host, numel, h->cfg.device, h->stream);
}

// ---- NCCL through dlopen (no link-time dependency: the library loads on machines without NCCL or a GPU)
struct NcclUniqueId { char b[128]; };
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, NcclUniqueId, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*CommSplit)(void*, int, int, void**, void*) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
extern NcclApi g_nccl;
int load_nccl(const char* path);
// 0 or a negative B2G_E* code with b2g_last_error() set
int nccl_comm_init(void** comm, int nranks, const void* id128, int rank, const char* lib);
int nccl_allreduce_sum_f32(void* comm, float* buf, size_t count, cudaStream_t s);
void nccl_comm_destroy(void* comm);

}  // namespace b2g
