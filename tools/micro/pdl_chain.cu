// Micro-benchmark: what does programmatic dependent launch buy for a chain of short dependent kernels inside a CUDA graph?
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pdl_chain pdl_chain.cu && ./pdl_chain
// Kernel = one CTA per SM x 256 threads, SMEM bytes of dynamic shared memory (1 CTA / SM when large), prologue (barrier-init stand-in),
// then a streaming read-modify-write of `elems` floats (dependent on the previous kernel's output).
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>

__global__ void __launch_bounds__(256, 1) body(const float* __restrict__ in, float* __restrict__ out, int elems, int pdl) {
  extern __shared__ float sm[];
  sm[threadIdx.x] = (float)threadIdx.x;              // prologue stand-in
  __syncthreads();
  if (pdl) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
  }
  float acc = sm[(threadIdx.x + 1) & 255] * 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < elems; i += gridDim.x * blockDim.x) out[i] = in[i] * 1.0001f + acc;
}

static float run(int n_kernels, int smem, int elems, int pdl, int threads_grid) {
  float *a, *b;
  cudaMalloc(&a, elems * 4); cudaMalloc(&b, elems * 4);
  cudaMemset(a, 0, elems * 4); cudaMemset(b, 0, elems * 4);
  cudaFuncSetAttribute(body, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaStream_t s; cudaStreamCreate(&s);
  cudaGraph_t g; cudaGraphExec_t ge;
  cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal);
  for (int k = 0; k < n_kernels; ++k) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(threads_grid); cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
    const float* in = (k & 1) ? b : a; float* out = (k & 1) ? a : b;
    cudaError_t e = cudaLaunchKernelEx(&cfg, body, in, out, elems, pdl);
    if (e != cudaSuccess) { printf("launch error %s\n", cudaGetErrorString(e)); exit(1); }
  }
  cudaError_t e = cudaStreamEndCapture(s, &g);
  if (e != cudaSuccess) { printf("capture error %s\n", cudaGetErrorString(e)); exit(1); }
  e = cudaGraphInstantiate(&ge, g, 0);
  if (e != cudaSuccess) { printf("instantiate error %s\n", cudaGetErrorString(e)); exit(1); }
  for (int i = 0; i < 3; ++i) cudaGraphLaunch(ge, s);
  cudaStreamSynchronize(s);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0, s);
  for (int i = 0; i < 10; ++i) cudaGraphLaunch(ge, s);
  cudaEventRecord(e1, s);
  cudaStreamSynchronize(s);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  e = cudaGetLastError();
  if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); exit(1); }
  cudaFree(a); cudaFree(b);
  return ms * 1000.f / (10 * n_kernels);
}

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  const int smems[2] = {1024, 200 * 1024};
  const int elems[3] = {1 << 16, 1 << 21, 1 << 23};       // 0.25 MB, 8 MB, 32 MB per tensor
  for (int si = 0; si < 2; ++si)
    for (int ei = 0; ei < 3; ++ei) {
      float t0 = run(200, smems[si], elems[ei], 0, sms);
      float t1 = run(200, smems[si], elems[ei], 1, sms);
      printf("smem %6d B  tensor %5.2f MB : %.2f us/kernel plain, %.2f us/kernel PDL\n", smems[si], elems[ei] * 4 / 1e6, t0, t1);
    }
  return 0;
}
