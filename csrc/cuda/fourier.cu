// K4: PS-side decode of the cyclic (Fourier) gradient code.
//
// Reference flow per parameter tensor (src/master/cyclic_master.py:152-173 + src/c_coding.cpp): E = R f
// (numpy complex128 dot over d), locator solve in C++/Eigen, healthy-row pick, scipy lsq_linear for the
// recombination vector v, then decoded = v^T R and Re(.)/n.  The two passes over the n x d matrix R are the
// heavy part; everything else is O(n^3) per tensor.
//
// Device formulation: (a) `cyclic_project_kernel`: one streaming pass over the complex64 arena R[n][D]
// producing per-tile partials with fp64 accumulation, folded per tensor in a fixed order by `cyclic_fold_kernel`
// (E[T][n]; no atomics -> the decode is bit-reproducible);
// (b) `cyclic_locate_kernel`: one CTA per tensor (lane 0 of one warp) runs the shared fp64 locator core
// (csrc/common/locator_core.h) and emits v[T][n] as complex64; (c) the recombination Re(v^T R)/n is fused
// with SGD + broadcast in aggregate_update.cu (mode 1).  No host round trip between (a), (b) and (c).
#include "common.cuh"
#include "../common/locator_core.h"

struct ProjectArgs {
  const float* R;                 // [n][2*slot_stride] complex64 interleaved
  long long slot_stride;          // complex elements per worker slot
  int n;
  const float* f;                 // [D] random projection factors (N(1,1), fixed at build time)
  TileView tv;
  double* E;                      // [T][n][2] (re, im): per-tensor totals, written by the fold kernel
  double* Epart;                  // [ntiles][n][2] per-tile partials (workspace)
};

// Pass 1: every tile's contribution E_tile[i] = sum_d R_i[d] f[d] for all n workers at once (all loads of a tile issued up
// front, ONE block reduction per tile) -> Epart.  No atomics: the summation order is fixed, so the decode is bit-reproducible.
__global__ void __launch_bounds__(DRC_THREADS) cyclic_project_kernel(const __grid_constant__ ProjectArgs a) {
  __shared__ double s_part[DRC_THREADS / 32][2 * DRC_MAX_R];
  for (int tile = blockIdx.x; tile < a.tv.ntiles; tile += gridDim.x) {
    int tensor;
    const int valid = tile_valid(a.tv, tile, tensor);
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    const bool active = (int)threadIdx.x * 4 < valid;
    float4 f4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (active) f4 = *reinterpret_cast<const float4*>(a.f + idx);
    for (int i0 = 0; i0 < a.n; i0 += DRC_MAX_R) {             // workers in chunks of 8 (16 fp64 accumulators per thread)
      double acc[2 * DRC_MAX_R];
#pragma unroll
      for (int ii = 0; ii < DRC_MAX_R; ++ii) {
        const int i = i0 + ii;
        double re = 0.0, im = 0.0;
        if (i < a.n && active) {
          const float4* src = reinterpret_cast<const float4*>(a.R + 2 * (i * a.slot_stride + idx));
          float4 c0 = ld_f4(src), c1 = ld_f4(src + 1);
          re = (double)c0.x * f4.x + (double)c0.z * f4.y + (double)c1.x * f4.z + (double)c1.z * f4.w;
          im = (double)c0.y * f4.x + (double)c0.w * f4.y + (double)c1.y * f4.z + (double)c1.w * f4.w;
        }
        acc[2 * ii] = re; acc[2 * ii + 1] = im;
      }
      const int nj = 2 * (a.n - i0 < DRC_MAX_R ? a.n - i0 : DRC_MAX_R);
#pragma unroll
      for (int j = 0; j < 2 * DRC_MAX_R; ++j) {
        if (j < nj) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
          if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5][j] = acc[j];
        }
      }
      __syncthreads();
      if ((int)threadIdx.x < nj) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < DRC_THREADS / 32; ++w) t += s_part[w][threadIdx.x];
        a.Epart[(long long)tile * 2 * a.n + 2 * i0 + threadIdx.x] = t;
      }
      __syncthreads();
    }
  }
}

// Pass 2: one warp per tensor folds its tiles' partials in a fixed order (lanes stride over the tiles, xor tree) -> E[T][n][2].
__global__ void __launch_bounds__(32) cyclic_fold_kernel(const __grid_constant__ ProjectArgs a) {
  const int t = blockIdx.x;
  const TensorMeta m = a.tv.meta[t];
  const long long tile0 = m.offset / DRC_TILE, ntile = (m.numel + DRC_TILE - 1) / DRC_TILE;
  for (int j = 0; j < 2 * a.n; ++j) {
    double s = 0.0;
    for (long long q = threadIdx.x; q < ntile; q += 32) s += a.Epart[(tile0 + q) * 2 * a.n + j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) a.E[(long long)t * 2 * a.n + j] = s;
  }
}

extern "C" int drc_cyclic_project(const ProjectArgs* args, int grid, cudaStream_t stream) {
  cyclic_project_kernel<<<grid, DRC_THREADS, 0, stream>>>(*args);
  cyclic_fold_kernel<<<args->tv.ntensors, 32, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}

struct LocateArgs {
  double* E;                      // [T][n][2]; zeroed after use (kept from the accumulate-in-place version; harmless)
  int T, n, s;
  double rel_tol;
  float2* recomb;                 // [T][n] out
  unsigned int* healthy;          // [T] out bitmask of rows used
  int* flagged;                   // [T] out number of rows flagged Byzantine
};

// One CTA per tensor: the locator is a serial O(n^3) fp64 computation per tensor, so the only parallelism is ACROSS tensors -- and
// the chain is latency-bound, so the tensors are spread over as many SMs as there are tensors (62 CTAs for ResNet-18) instead of
// sharing the fp64 pipe of two SMs (one warp per 32 tensors).
__global__ void __launch_bounds__(32) cyclic_locate_kernel(const __grid_constant__ LocateArgs a) {
  const int t = blockIdx.x;
  if (threadIdx.x != 0 || t >= a.T) return;
  cplx E[DRC_LOC_MAX_N], v[DRC_LOC_MAX_N];
  for (int i = 0; i < a.n; ++i) {
    E[i] = c_make(a.E[((long long)t * a.n + i) * 2], a.E[((long long)t * a.n + i) * 2 + 1]);
    a.E[((long long)t * a.n + i) * 2] = 0.0;
    a.E[((long long)t * a.n + i) * 2 + 1] = 0.0;
  }
  unsigned int mask = 0u;
  int fl = locate_and_recombine(E, a.n, a.s, a.rel_tol, v, &mask);
  for (int i = 0; i < a.n; ++i) a.recomb[(long long)t * a.n + i] = make_float2((float)v[i].re, (float)v[i].im);
  if (a.healthy) a.healthy[t] = mask;
  if (a.flagged) a.flagged[t] = fl;
}

extern "C" int drc_cyclic_locate(const LocateArgs* args, cudaStream_t stream) {
  if (args->n > DRC_LOC_MAX_N || args->s > DRC_LOC_MAX_S) return (int)cudaErrorInvalidValue;
  cyclic_locate_kernel<<<args->T, 32, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}

extern "C" int drc_sizeof_ProjectArgs() { return (int)sizeof(ProjectArgs); }
extern "C" int drc_sizeof_LocateArgs() { return (int)sizeof(LocateArgs); }
