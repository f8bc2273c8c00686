// Per-edge latency of a captured chain of dependent kernels, with and without programmatic
// dependent launch. build: nvcc -gencode arch=compute_90a,code=sm_90a -o pdl_probe pdl_probe.cu
#include <cstdio>
#include <cuda_runtime.h>
#include <vector>
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s:%d %s -> %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); fflush(stdout); return -1.f; } } while (0)

template <bool PDL>
__global__ void __launch_bounds__(640, 1) chain_kernel(float* p, int spin, int smem_touch) {
  extern __shared__ float sm[];
  // "prologue": touch shared memory like a barrier/descriptor set-up would
  for (int i = threadIdx.x; i < smem_touch; i += blockDim.x) sm[i] = 0.f;
  __syncthreads();
  if (PDL) asm volatile("griddepcontrol.wait;" ::: "memory");
  float v = p[blockIdx.x * blockDim.x + threadIdx.x];
  long long t0 = clock64();
  while (clock64() - t0 < spin) v += 1e-9f;
  p[blockIdx.x * blockDim.x + threadIdx.x] = v + (smem_touch > 0 ? sm[threadIdx.x % smem_touch] : 0.f);
}

template <bool PDL>
float run(int nk, int grid, int spin, size_t smem, int reps) {
  float* p;
  CK(cudaMalloc(&p, sizeof(float) * 640 * 1024));
  cudaMemset(p, 0, sizeof(float) * 640 * 1024);
  cudaStream_t s;
  CK(cudaStreamCreate(&s));
  if (smem > 0) CK(cudaFuncSetAttribute(chain_kernel<PDL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaGraph_t g = nullptr;
  cudaGraphExec_t ge = nullptr;
  CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
  for (int i = 0; i < nk; ++i) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(640);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = (PDL && i > 0) ? 1 : 0;
    int st = (int)(smem / 4 > 4096 ? 4096 : smem / 4);
    CK(cudaLaunchKernelEx(&cfg, chain_kernel<PDL>, p, spin, st));
  }
  CK(cudaStreamEndCapture(s, &g));
  cudaError_t e = cudaGraphInstantiate(&ge, g, 0);
  if (e != cudaSuccess) { printf("instantiate: %s\n", cudaGetErrorString(e)); return -1; }
  for (int i = 0; i < 5; ++i) cudaGraphLaunch(ge, s);
  cudaStreamSynchronize(s);
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  cudaEventRecord(a, s);
  for (int i = 0; i < reps; ++i) cudaGraphLaunch(ge, s);
  cudaEventRecord(b, s);
  cudaStreamSynchronize(s);
  float ms;
  cudaEventElapsedTime(&ms, a, b);
  e = cudaGetLastError();
  if (e != cudaSuccess) printf("error: %s\n", cudaGetErrorString(e));
  cudaFree(p);
  return ms * 1000.f / reps;
}

int main() {
  const int nk = 13;
  for (int spin : {0, 20000, 100000}) {
    for (size_t smem : {(size_t)0, (size_t)200 * 1024}) {
      for (int grid : {16, 148, 592}) {
        float a = run<false>(nk, grid, spin, smem, 200);
        float b = run<true>(nk, grid, spin, smem, 200);
        printf("spin %6d cyc smem %3zu KB grid %3d: plain %.2f us/graph (%.2f/kernel)  PDL %.2f us/graph (%.2f/kernel)\n",
               spin, smem >> 10, grid, a, a / nk, b, b / nk);
      }
    }
  }
  return 0;
}
