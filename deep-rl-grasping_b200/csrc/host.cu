// libb200grasp: host runtime shared by the learner and encoder handles (declarations and contracts in host.cuh), and the
// library-wide part of the C ABI.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "host.cuh"

thread_local std::string g_b2g_err;
int b2g_fail(int code, const std::string& msg) { g_b2g_err = msg; return code; }

namespace b2g {

int check_device(int device, int* num_sms) {
  int ndev = 0;
  CK(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return b2g_fail(B2G_ECUDA, "no such CUDA device");
  CK(cudaSetDevice(device));
  cudaDeviceProp prop{};
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9) return b2g_fail(B2G_ECUDA, std::string("libb200grasp is built for sm_90a only; found ") + prop.name);
  if (num_sms) *num_sms = prop.multiProcessorCount;
  return 0;
}

int upload_table(std::vector<void*>& allocs, cudaStream_t s, const std::vector<int>& v, const int** out,
                 std::map<const int*, std::vector<int>>* host_copy) {
  int* d = nullptr;
  if (int rc = dev_alloc(allocs, s, &d, v.size(), false)) return rc;
  CK(cudaMemcpyAsync(d, v.data(), v.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  CK(cudaStreamSynchronize(s));
  *out = d;
  if (host_copy) (*host_copy)[d] = v;
  return 0;
}

std::vector<int> iota_tab(int n, int stride, int base) {
  std::vector<int> v(n);
  for (int i = 0; i < n; ++i) v[i] = base + i * stride;
  return v;
}

GemmDesc gemm_desc(const float* A, const int* aM, const int* aR, const float* B, const int* bR, const int* bN, float* C,
                   const int* cM, const int* cN, int M, int N, int R, int flags, int splitR) {
  GemmDesc d{};
  d.A = A; d.B = B; d.C = C; d.aM = aM; d.aR = aR; d.bR = bR; d.bN = bN; d.cM = cM; d.cN = cN;
  d.M = M; d.N = N; d.R = R; d.flags = flags; d.splitR = splitR; d.alpha = 1.f;
  return d;
}

int finalize_tiles(GemmGroup& g, std::vector<void*>& allocs, cudaStream_t s, int bm, int bn) {
  int start = 0;
  for (auto& d : g.host) {
    d.tiles_m = (d.M + bm - 1) / bm;
    d.tiles_n = (d.N + bn - 1) / bn;
    d.tile_start = start;
    d.tile_count = d.tiles_m * d.tiles_n * d.splitR;
    start += d.tile_count;
  }
  g.total_tiles = start;
  if (!g.dev)
    if (int rc = dev_alloc(allocs, s, &g.dev, g.host.size(), false)) return rc;
  CK(cudaMemcpyAsync(g.dev, g.host.data(), g.host.size() * sizeof(GemmDesc), cudaMemcpyHostToDevice, s));
  CK(cudaStreamSynchronize(s));     // g.host is pageable
  return 0;
}

void gg_tc_columns(GemmDesc& d, const std::map<const int*, std::vector<int>>& host_tabs, ColIds& col_ids) {
  {   // GG_CN_AFFINE4: column tables contiguous in aligned groups of 4, row offsets multiples of 4
    auto grp4 = [&](const int* tab, int n) {
      auto it = host_tabs.find(tab);
      if (it == host_tabs.end() || (int)it->second.size() < n) return false;
      const std::vector<int>& v = it->second;
      for (int i = 0; i + 3 < n; i += 4)
        if ((v[i] & 3) || v[i + 1] != v[i] + 1 || v[i + 2] != v[i] + 2 || v[i + 3] != v[i] + 3) return false;
      return true;
    };
    auto mult4 = [&](const int* tab, int n) {
      auto it = host_tabs.find(tab);
      if (it == host_tabs.end() || (int)it->second.size() < n) return false;
      for (int i = 0; i < n; ++i) if (it->second[i] & 3) return false;
      return true;
    };
    bool ok = (d.N % 4 == 0) && grp4(d.cN, d.N) && mult4(d.cM, d.M);
    if (ok && (d.flags & (GG_EPI_MASK | GG_EPI_LRELU_GRAD))) ok = (!d.kN || grp4(d.kN, d.N)) && (!d.kM || mult4(d.kM, d.M));
    if (ok) d.flags |= GG_CN_AFFINE4;
  }
  {   // column-table identity (gg_tc.cu epilogue): descriptors with the same tables never trigger a re-stage
    const auto key = std::make_tuple((const void*)d.cN, (const void*)d.kN,
                                     (const void*)((d.flags & GG_EPI_BIAS_RELU) ? d.bias : nullptr), d.N);
    auto it = col_ids.find(key);
    if (it == col_ids.end()) it = col_ids.emplace(key, (int)col_ids.size()).first;
    d.col_id = it->second;
  }
}

int capture_graph(cudaStream_t s, const std::function<int()>& issue, cudaGraphExec_t* exec) {
  cudaGraph_t graph = nullptr;
  CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
  const int rc = issue();
  const cudaError_t e = cudaStreamEndCapture(s, &graph);
  if (rc || e != cudaSuccess) {
    if (graph) cudaGraphDestroy(graph);
    return rc ? rc : b2g_fail(B2G_ECUDA, std::string("graph capture failed: ") + cudaGetErrorString(e));
  }
  const cudaError_t e2 = cudaGraphInstantiate(exec, graph, 0);
  cudaGraphDestroy(graph);
  if (e2 != cudaSuccess) return b2g_fail(B2G_ECUDA, std::string("graph instantiate failed: ") + cudaGetErrorString(e2));
  return 0;
}

int upload_lr(float* d_lr, float* cur_lr, float lr, cudaStream_t s) {
  if (lr != *cur_lr) {
    CK(cudaStreamSynchronize(s));
    CK(cudaMemcpy(d_lr, &lr, sizeof(float), cudaMemcpyHostToDevice));
    *cur_lr = lr;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------ named parameters
void ParamTable::add(const std::string& name, int64_t rows, int64_t cols, int ndim, int stride, int64_t off, bool grad) {
  index_[name] = (int)entries_.size();
  entries_.push_back(ParamEntry{name, rows, cols, ndim, stride, off, grad, nullptr});
}

void ParamTable::add_scalar(const std::string& name, float* v) {
  index_[name] = (int)entries_.size();
  entries_.push_back(ParamEntry{name, 1, 1, 0, 1, -1, false, v});
}

void ParamTable::add_copies(int first, int n, const std::string& from_scope, const std::string& to_scope, int64_t shift) {
  for (int i = first; i < first + n; ++i) {
    const ParamEntry e = entries_[i];
    add(to_scope + e.name.substr(from_scope.size()), e.rows, e.cols, e.ndim, e.stride, e.off + shift, false);
  }
}

int ParamTable::info(int idx, char* name, size_t name_cap, int64_t* rows, int64_t* cols, int32_t* ndim) const {
  if (idx < 0 || idx >= count() || !name) return b2g_fail(B2G_EINVAL, "bad tensor index");
  const ParamEntry& e = entries_[idx];
  snprintf(name, name_cap, "%s", e.name.c_str());
  if (rows) *rows = e.rows;
  if (cols) *cols = e.cols;
  if (ndim) *ndim = e.ndim;
  return 0;
}

int ParamTable::copy(const char* name, ParamCopy mode, float* P, float* G, float* host, size_t numel, int device, cudaStream_t s) const {
  if (!name || !host) return b2g_fail(B2G_EINVAL, "NULL argument");
  std::string nm(name);
  if (nm.size() > 2 && nm.compare(nm.size() - 2, 2, ":0") == 0) nm.resize(nm.size() - 2);
  CK(cudaSetDevice(device));
  CK(cudaStreamSynchronize(s));
  const auto it = index_.find(nm);
  if (it == index_.end()) return b2g_fail(B2G_EINVAL, std::string("unknown variable: ") + name);
  const ParamEntry& e = entries_[it->second];
  if (numel != (size_t)(e.rows * e.cols)) return b2g_fail(B2G_EINVAL, std::string("size mismatch for ") + name);
  if (e.scalar) {
    if (mode == ParamCopy::Set) *e.scalar = host[0];
    else host[0] = *e.scalar;
    return 0;
  }
  if (mode == ParamCopy::GetGrad && !e.grad) return b2g_fail(B2G_EINVAL, std::string("no gradient for ") + name);
  float* dev = (mode == ParamCopy::GetGrad ? G : P) + e.off;
  const size_t row = e.cols * sizeof(float), pitch = e.stride * sizeof(float);
  if (mode == ParamCopy::Set) CK(cudaMemcpy2D(dev, pitch, host, row, row, e.rows, cudaMemcpyHostToDevice));
  else CK(cudaMemcpy2D(host, row, dev, pitch, row, e.rows, cudaMemcpyDeviceToHost));
  return 0;
}

// ------------------------------------------------------------------------------------------------ NCCL
NcclApi g_nccl;

int load_nccl(const char* path) {
  if (g_nccl.lib) return 0;
  const char* cands[] = {path, "libnccl.so.2", "libnccl.so", "/usr/lib/x86_64-linux-gnu/libnccl.so.2"};
  for (const char* c : cands) {
    if (!c || !*c) continue;
    g_nccl.lib = dlopen(c, RTLD_NOW | RTLD_GLOBAL);
    if (g_nccl.lib) break;
  }
  if (!g_nccl.lib) return b2g_fail(B2G_ENCCL, std::string("cannot dlopen libnccl: ") + dlerror());
  g_nccl.GetUniqueId = (int (*)(void*))dlsym(g_nccl.lib, "ncclGetUniqueId");
  g_nccl.CommInitRank = (int (*)(void**, int, NcclUniqueId, int))dlsym(g_nccl.lib, "ncclCommInitRank");
  g_nccl.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(g_nccl.lib, "ncclAllReduce");
  g_nccl.CommDestroy = (int (*)(void*))dlsym(g_nccl.lib, "ncclCommDestroy");
  g_nccl.GetErrorString = (const char* (*)(int))dlsym(g_nccl.lib, "ncclGetErrorString");
  g_nccl.CommSplit = (int (*)(void*, int, int, void**, void*))dlsym(g_nccl.lib, "ncclCommSplit");
  g_nccl.GroupStart = (int (*)())dlsym(g_nccl.lib, "ncclGroupStart");
  g_nccl.GroupEnd = (int (*)())dlsym(g_nccl.lib, "ncclGroupEnd");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce)
    return b2g_fail(B2G_ENCCL, "libnccl is missing symbols");
  return 0;
}

int nccl_comm_init(void** comm, int nranks, const void* id128, int rank, const char* lib) {
  if (int rc = load_nccl(lib)) return rc;
  NcclUniqueId id;
  memcpy(id.b, id128, 128);
  // (B2G_AR_SMS also caps NCCL's CTAs: a collective that overlaps the persistent GEMM grids -- one CTA per SM, 226 KB of shared
  //  memory each, nothing fits beside them -- displaces every GEMM CTA beyond the reserve.  Measured at N = 2: capping at 8 CTAs
  //  halves the all-reduce bandwidth and costs more than it saves, so the cap is opt-in.)
  if (!getenv("NCCL_MAX_CTAS")) { if (const char* e = getenv("B2G_AR_SMS")) setenv("NCCL_MAX_CTAS", e, 0); }
  const int nrc = g_nccl.CommInitRank(comm, nranks, id, rank);
  if (nrc != 0) return b2g_fail(B2G_ENCCL, std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(nrc) : "?"));
  return 0;
}
int nccl_allreduce_sum_f32(void* comm, float* buf, size_t count, cudaStream_t s) {
  const int nrc = g_nccl.AllReduce(buf, buf, count, /*ncclFloat32*/ 7, /*ncclSum*/ 0, comm, s);
  if (nrc != 0) return b2g_fail(B2G_ENCCL, std::string("ncclAllReduce: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(nrc) : "?"));
  return 0;
}
void nccl_comm_destroy(void* comm) { if (comm && g_nccl.CommDestroy) g_nccl.CommDestroy(comm); }

}  // namespace b2g

using namespace b2g;

extern "C" {

const char* b2g_last_error(void) { return g_b2g_err.c_str(); }
int b2g_version(void) { return 100; }

int b2g_nccl_unique_id(void* out128, const char* nccl_lib) {
  if (!out128) return b2g_fail(B2G_EINVAL, "out128 is NULL");
  if (int rc = load_nccl(nccl_lib)) return rc;
  int rc = g_nccl.GetUniqueId(out128);
  if (rc != 0) return b2g_fail(B2G_ENCCL, "ncclGetUniqueId failed");
  return 0;
}

}  // extern "C"
