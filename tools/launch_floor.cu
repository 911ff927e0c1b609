// launch_floor: what does ONE dependent launch of a persistent 1-CTA/SM kernel cost inside a CUDA graph on this GPU?
// Variants: plain empty kernel; + 200 KiB dynamic shared memory; + programmatic dependent launch;
// alternating big-smem / small-smem kernels (shared-memory carve-out switches).  Prints microseconds per launch.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O2 -o tools/launch_floor tools/launch_floor.cu
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at line %d\n", cudaGetErrorString(e_), __LINE__); exit(2); } } while (0)

__global__ void __launch_bounds__(320, 1) k_big(int pdl, float* sink) {
  extern __shared__ unsigned char smem[];
  if (pdl) { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); asm volatile("griddepcontrol.wait;" ::: "memory"); }
  if (sink && threadIdx.x == 0 && blockIdx.x == 0) sink[0] += 1.f;
}
__global__ void k_small(float* sink) { if (sink && threadIdx.x == 0 && blockIdx.x == 0) sink[0] += 1.f; }

static float run(int nl, int sms, int smem, int pdl, int alternate, float* sink) {
  cudaStream_t s; CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  cudaGraph_t g; cudaGraphExec_t ge;
  CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
  for (int i = 0; i < nl; ++i) {
    if (alternate && (i & 1)) { k_small<<<256, 256, 0, s>>>(sink); continue; }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(sms); cfg.blockDim = dim3(320); cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
    CK(cudaLaunchKernelEx(&cfg, k_big, pdl, sink));
  }
  CK(cudaStreamEndCapture(s, &g));
  CK(cudaGraphInstantiate(&ge, g, 0));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  for (int w = 0; w < 5; ++w) CK(cudaGraphLaunch(ge, s));
  CK(cudaEventRecord(e0, s));
  const int reps = 50;
  for (int r = 0; r < reps; ++r) CK(cudaGraphLaunch(ge, s));
  CK(cudaEventRecord(e1, s));
  CK(cudaStreamSynchronize(s));
  float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
  cudaGraphExecDestroy(ge); cudaGraphDestroy(g); cudaStreamDestroy(s);
  return ms * 1e3f / (reps * nl);
}

int main() {
  float* sink; CK(cudaMalloc(&sink, 4)); CK(cudaMemset(sink, 0, 4));
  CK(cudaFuncSetAttribute(k_big, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
  int dev = 0, sms = 0;
  CK(cudaGetDevice(&dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int nl = 20;
  printf("empty %dx320, no smem             : %.2f us / launch\n", sms, run(nl, sms, 0, 0, 0, sink));
  printf("empty %dx320, 200 KiB smem        : %.2f us / launch\n", sms, run(nl, sms, 200 * 1024, 0, 0, sink));
  printf("  + PDL                           : %.2f us / launch\n", run(nl, sms, 200 * 1024, 1, 0, sink));
  printf("alternating 200 KiB / small kernel: %.2f us / launch\n", run(nl, sms, 200 * 1024, 0, 1, sink));
  printf("alternating, PDL on big           : %.2f us / launch\n", run(nl, sms, 200 * 1024, 1, 1, sink));
  return 0;
}
