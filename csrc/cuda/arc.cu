// Adaptive robust clipping (ARC; Allouah, Guerraoui, Gupta, Jellouli, Rizk and Stephan, arXiv 2405.14432) on the P raw worker
// slots, after the PS-side attack and before the row source and the base rule (codes/oracle.py::arc holds the semantics).  With
// k = floor(2 f (P - f) / P), per tensor (or once over the whole model):
//
//   arc_norm_kernel     d_i = sum_e (double)x_ie^2 as per-tile fp64 partials [ntiles][P] (cc_dist_kernel's order, no centre)
//   arc_factors_kernel  the partials of each tensor folded in tile order; d_tau = the (k+1)-th largest d_i (NaN largest);
//                       a_i = 1 when !(d_i > d_tau), else fp32(sqrt(d_tau) / sqrt(d_i)) formed in fp64
//   arc_scale_kernel    x_i <- x_i * a_i (one fp32 multiply) in place, only for the rows with a_i < 1
//
// With --arc model, clip.cu's cc_fold_kernel (drc_cc_fold) folds the partials per tensor into dist[T][P] and
// arc_model_factors_kernel sums them over the tensors in ascending order and writes one factor row into all T rows.
//
// Determinism: per-thread sums, warp shuffles in a fixed pattern, the 8 warps in order, then the fold in tile order.  No
// floating-point atomics: the factors and the slab depend neither on the grid nor on how the arena is cut into buckets.
#include "common.cuh"

#define ARC_MAXP 16                                               // = ROBUST_MAXP: the rows live in registers
#define ARC_FOLD 32                                               // = CC_FOLD: tiles whose partials are loaded together

struct ArcArgs {
  float* grad_in;                         // [P][slot_stride] worker slots (PS memory), clipped in place
  long long slot_stride;
  int P;
  int k;                                  // rows clipped: floor(2 f (P - f) / P)
  TileView tv;
  double* partials;                       // [ntiles][P]
  float* factors;                         // [T][P]
  const double* dist;                     // model scope: [T][P] the per-tensor d_i (drc_cc_fold)
  int tile_begin, tile_end;               // norm / scale: tiles (tile_end == 0: to the end of the arena)
  int t_begin, t_end;                     // factors: tensors (t_end == 0: every tensor); buckets hold whole tensors
};

__global__ void __launch_bounds__(DRC_THREADS) arc_norm_kernel(const __grid_constant__ ArcArgs a) {
  __shared__ double s_part[DRC_THREADS / 32][ARC_MAXP];
  const int P = a.P;
  const int tile_end = a.tile_end > 0 ? a.tile_end : a.tv.ntiles;
  for (int tile = a.tile_begin + blockIdx.x; tile < tile_end; tile += gridDim.x) {
    int tensor;
    const int valid = tile_valid(a.tv, tile, tensor);
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    const int lane_valid = valid - (int)threadIdx.x * 4;        // real elements of this thread (<= 0: padding only)
    float4 x[ARC_MAXP];
#pragma unroll
    for (int i = 0; i < ARC_MAXP; ++i) {
      x[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (i < P && lane_valid > 0) x[i] = ld_f4(reinterpret_cast<const float4*>(a.grad_in + i * a.slot_stride + idx));
    }
#pragma unroll
    for (int i = 0; i < ARC_MAXP; ++i) {
      if (i < P) {
        double d = 0.0;
        if (lane_valid > 0) {
          const double e0 = (double)x[i].x;
          d = __dmul_rn(e0, e0);
          if (lane_valid > 1) { const double e = (double)x[i].y; d = __dadd_rn(d, __dmul_rn(e, e)); }
          if (lane_valid > 2) { const double e = (double)x[i].z; d = __dadd_rn(d, __dmul_rn(e, e)); }
          if (lane_valid > 3) { const double e = (double)x[i].w; d = __dadd_rn(d, __dmul_rn(e, e)); }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) d = __dadd_rn(d, __shfl_xor_sync(0xffffffffu, d, o));
        if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5][i] = d;
      }
    }
    __syncthreads();
    if ((int)threadIdx.x < P) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < DRC_THREADS / 32; ++w) s = __dadd_rn(s, s_part[w][threadIdx.x]);
      a.partials[(long long)tile * P + threadIdx.x] = s;
    }
    __syncthreads();
  }
}

// d ranks above e: the larger value, a NaN above every number
__device__ __forceinline__ bool arc_above(double d, double e) { return (isnan(d) && !isnan(e)) || d > e; }

// Lane i < P of a full warp holds d_i; every lane returns a_i (lanes >= P: 1).  d_tau is the value of the lane of rank k, the
// rank of lane i being the lanes above it plus the equal lanes below it, so exactly one lane has each rank
__device__ __forceinline__ float arc_factor(double d, int P, int k) {
  const int i = threadIdx.x & 31;
  int rank = 0;
  for (int j = 0; j < P; ++j) {
    const double e = __shfl_sync(0xffffffffu, d, j);
    rank += (arc_above(e, d) || (j < i && !arc_above(d, e))) ? 1 : 0;
  }
  const unsigned int at_k = __ballot_sync(0xffffffffu, i < P && rank == k);
  const double tau = __shfl_sync(0xffffffffu, d, __ffs(at_k) - 1);
  if (i >= P || !(d > tau)) return 1.f;
  return (float)__ddiv_rn(__dsqrt_rn(tau), __dsqrt_rn(d));
}

// one warp per tensor: lane i < P folds row i's partials over the tensor's tiles in tile order (cc_weights_kernel's fold)
__global__ void __launch_bounds__(DRC_THREADS) arc_factors_kernel(const __grid_constant__ ArcArgs a) {
  const int t_end = a.t_end > 0 ? a.t_end : a.tv.ntensors;
  const int tensor = a.t_begin + (int)(blockIdx.x * (DRC_THREADS / 32) + (threadIdx.x >> 5));
  const int i = threadIdx.x & 31, P = a.P;
  if (tensor >= t_end) return;                                   // whole warps: the rank count shuffles over all 32 lanes
  const TensorMeta m = a.tv.meta[tensor];
  const int t0 = (int)(m.offset / DRC_TILE), t1 = t0 + (int)((m.numel + DRC_TILE - 1) / DRC_TILE);
  double d = 0.0;
  if (i < P) {
    const double* p = a.partials + i;
    int t = t0;
    for (; t + ARC_FOLD <= t1; t += ARC_FOLD) {
      double b[ARC_FOLD];
#pragma unroll
      for (int q = 0; q < ARC_FOLD; ++q) b[q] = p[(long long)(t + q) * P];
#pragma unroll
      for (int q = 0; q < ARC_FOLD; ++q) d = __dadd_rn(d, b[q]);
    }
    for (; t < t1; ++t) d = __dadd_rn(d, p[(long long)t * P]);
  }
  const float f = arc_factor(d, P, a.k);
  if (i < P) a.factors[tensor * P + i] = f;
}

// one CTA: lane i of warp 0 sums dist[t][i] over t in ascending order (a NaN or Inf in one tensor reaches the sum), and the CTA
// writes the one factor row into all T rows
__global__ void __launch_bounds__(DRC_THREADS) arc_model_factors_kernel(const __grid_constant__ ArcArgs a) {
  __shared__ float s_f[ARC_MAXP];
  const int P = a.P, T = a.tv.ntensors;
  if (threadIdx.x < 32) {
    const int i = threadIdx.x;
    double d = 0.0;
    if (i < P) {
      int t = 0;
      for (; t + ARC_FOLD <= T; t += ARC_FOLD) {
        double b[ARC_FOLD];
#pragma unroll
        for (int q = 0; q < ARC_FOLD; ++q) b[q] = a.dist[(t + q) * P + i];
#pragma unroll
        for (int q = 0; q < ARC_FOLD; ++q) d = __dadd_rn(d, b[q]);
      }
      for (; t < T; ++t) d = __dadd_rn(d, a.dist[t * P + i]);
    }
    const float f = arc_factor(d, P, a.k);
    if (i < P) s_f[i] = f;
  }
  __syncthreads();
  for (int q = threadIdx.x; q < T * P; q += DRC_THREADS) a.factors[q] = s_f[q % P];
}

// per tile: the rows whose factor for the tile's tensor is below 1 are multiplied in place; the others are not touched
__global__ void __launch_bounds__(DRC_THREADS) arc_scale_kernel(const __grid_constant__ ArcArgs a) {
  const int P = a.P;
  const int tile_end = a.tile_end > 0 ? a.tile_end : a.tv.ntiles;
  for (int tile = a.tile_begin + blockIdx.x; tile < tile_end; tile += gridDim.x) {
    int tensor;
    const int valid = tile_valid(a.tv, tile, tensor);
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    const int lane_valid = valid - (int)threadIdx.x * 4;
    if (lane_valid <= 0) continue;
    for (int i = 0; i < P; ++i) {
      const float f = a.factors[tensor * P + i];
      if (!(f < 1.f)) continue;
      float* p = a.grad_in + i * a.slot_stride + idx;
      const float4 x = ld_f4(reinterpret_cast<const float4*>(p));
      const float r[4] = {__fmul_rn(x.x, f), __fmul_rn(x.y, f), __fmul_rn(x.z, f), __fmul_rn(x.w, f)};
      store_row(p, r, lane_valid);
    }
  }
}

static bool arc_shape_ok(const ArcArgs* a) {
  return a->P >= 1 && a->P <= ARC_MAXP && a->k >= 0 && a->k < a->P && a->tv.ntensors >= 1;
}
extern "C" int drc_arc_norm(const ArcArgs* args, int grid, cudaStream_t stream) {
  if (!arc_shape_ok(args) || !args->grad_in || !args->partials || grid < 1) return (int)cudaErrorInvalidValue;
  arc_norm_kernel<<<grid, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_arc_factors(const ArcArgs* args, cudaStream_t stream) {
  if (!arc_shape_ok(args) || !args->partials || !args->factors) return (int)cudaErrorInvalidValue;
  const int t_end = args->t_end > 0 ? args->t_end : args->tv.ntensors;
  if (args->t_begin < 0 || t_end <= args->t_begin || t_end > args->tv.ntensors) return (int)cudaErrorInvalidValue;
  const int warps = DRC_THREADS / 32;
  arc_factors_kernel<<<(t_end - args->t_begin + warps - 1) / warps, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_arc_model_factors(const ArcArgs* args, cudaStream_t stream) {
  if (!arc_shape_ok(args) || !args->dist || !args->factors) return (int)cudaErrorInvalidValue;
  arc_model_factors_kernel<<<1, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_arc_scale(const ArcArgs* args, int grid, cudaStream_t stream) {
  if (!arc_shape_ok(args) || !args->grad_in || !args->factors || grid < 1) return (int)cudaErrorInvalidValue;
  arc_scale_kernel<<<grid, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_sizeof_ArcArgs() { return (int)sizeof(ArcArgs); }
