// Shared device-side definitions for the draco_b200 step-path kernels (sm_90a only).
//
// Arena model: every rank keeps its parameters / gradients / momentum in flat arenas that share one
// element layout.  A tensor starts at a multiple of TILE elements and owns ceil(numel / TILE) tiles, so a
// CTA working on a tile knows which tensor it belongs to (the reference applies vote / Krum / median /
// Fourier decode per parameter tensor: src/master/rep_master.py:154-168).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define DRC_TILE 1024            // elements per tile = 256 threads x float4
#define DRC_THREADS 256
#define DRC_MAX_WORKERS 32       // adversary bitmaps are 32-bit
#define DRC_MAX_R 8              // max members per repetition group / max cyclic redundancy 2s+1
#define DRC_MAX_DST 16           // max unicast broadcast destinations

struct TensorMeta {
  long long offset;              // element offset of the tensor in every arena (multiple of DRC_TILE)
  long long numel;
  int is_bf16;                   // compute dtype of this tensor on workers (1: bf16 arena, 0: fp32 arena)
  int pad;
};

struct HyperParams {             // lives in device memory so a captured graph sees updates
  // 48 bytes, the size the launch plans have always carried.  Every "1 - x" coefficient is formed in fp64 and rounded once to
  // fp32, as the library optimizers and codes/oracle.py::worker_momentum_coefficients do (fp32 1.f - 0.999f is 1.29e-5 away
  // from fp32(0.001)): fp32(1 - dampening) on the host, fp32(1 - beta) in the kernel from the fp64 betas, which the Adam bias
  // corrections 1 - beta^t also take.
  float lr, momentum, weight_decay;
  float one_minus_dampening;     // fp32(1 - dampening), 1 - dampening formed in fp64 on the host
  int nesterov;
  int optimizer;                 // 0: SGD-momentum (optim/sgd_modified.py:53-88), 1: Adam, 2: AMSGrad (optim/adam_modified.py:32-92)
  double beta1;                  // fp64 Adam betas
  float eps;
  int pad;
  double beta2;
};

// ---------------------------------------------------------------------------------------------
// system-scope synchronisation primitives (flags live in the *waiter's* memory; producers store remotely)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void fence_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }

// 16-byte streaming accesses.  Gradients are read once -> keep them out of L1; peer stores bypass L1 anyway.
__device__ __forceinline__ float4 ld_stream_f4(const float4* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ float4 ld_f4(const float4* p) {   // coherent (data written by peers this step)
  float4 v;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_f4(float4* p, float4 v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w) : "memory");
}
// one float4 of a slot row written in place; the tail of a tensor is stored element by element so that padding is never written
__device__ __forceinline__ void store_row(float* p, const float r[4], int lane_valid) {
  if (lane_valid >= 4) { st_f4(reinterpret_cast<float4*>(p), make_float4(r[0], r[1], r[2], r[3])); return; }
  p[0] = r[0];
  if (lane_valid > 1) p[1] = r[1];
  if (lane_valid > 2) p[2] = r[2];
}
// NVLS: one store, replicated by the NVSwitch into every GPU bound to the multicast object.
__device__ __forceinline__ void multimem_st_f4(float4* mc, float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w) : "memory");
}

__device__ __forceinline__ float4 bf16x4_to_f4(uint2 raw) {
  __nv_bfloat162 lo = *reinterpret_cast<__nv_bfloat162*>(&raw.x);
  __nv_bfloat162 hi = *reinterpret_cast<__nv_bfloat162*>(&raw.y);
  float2 a = __bfloat1622float2(lo), b = __bfloat1622float2(hi);
  return make_float4(a.x, a.y, b.x, b.y);
}

// ---------------------------------------------------------------------------------------------
// "last CTA" grid completion: returns true in exactly one CTA (all threads) after every CTA's prior
// global/peer writes are visible system-wide.  `counter` must be zero at launch; it is reset for reuse.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool grid_last_cta(unsigned int* counter) {
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    fence_sys();
    unsigned int prev = atomicAdd(counter, 1u);
    s_last = (prev == gridDim.x * gridDim.y - 1);
    if (s_last) { *counter = 0; fence_sys(); }
  }
  __syncthreads();
  return s_last != 0;
}

struct FlagList {                // flags to raise on completion (peer or local addresses)
  unsigned long long* ptr[DRC_MAX_DST];
  int n;
};

struct TileView {
  const int* tile_tensor;        // [ntiles] tensor id of each tile
  const TensorMeta* meta;        // [ntensors]
  int ntiles;
  int ntensors;
};

// number of valid elements of tile `tile` (0 < v <= DRC_TILE) and its tensor id
__device__ __forceinline__ int tile_valid(const TileView& tv, int tile, int& tensor) {
  tensor = tv.tile_tensor[tile];
  const TensorMeta m = tv.meta[tensor];
  long long start = (long long)tile * DRC_TILE - m.offset;
  long long left = m.numel - start;
  return left >= DRC_TILE ? DRC_TILE : (int)left;
}

#define DRC_CHECK_LAUNCH() (cudaGetLastError())
