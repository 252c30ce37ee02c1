// Centered clipping (Karimireddy, He and Jaggi, ICML 2021), one iteration per step around the previous aggregate
// (codes/oracle.py::centered_clip holds the semantics).  Per tensor, with the n <= CC_MAXP rows x_i, the centre v and tau:
//
//   cc_dist_kernel     d_i = sum_e ((double)x_ie - (double)v_e)^2 as per-tile fp64 partials [ntiles][n]
//   cc_weights_kernel  the partials of each tensor folded in tile order; w_i = fp32(min(1, tau / sqrt(d_i)) / n), 0 for a NaN
//                      or +Inf d_i
//   aggregate_update   mode 5: g = v + sum_i w_i (x_i - v), v <- g, then the optimizer (aggregate_update.cu)
//
// With --rule-scope model the norm is the whole model's: cc_fold_kernel + cc_model_weights_kernel replace cc_weights_kernel.
//
// The centre is last step's aggregate, known before the step starts, so only the n row-to-centre distances are needed: the
// rule runs bucket by bucket on the pipelined PS.  Rows come through an optional [n][T] row table (DETOX's winner_slot).
// Determinism: per-thread sums, warp shuffles in a fixed pattern, then the 8 warps in order into one partial per (tile, row),
// folded in tile order by the weights kernel.  No floating-point atomics: the weights depend neither on the grid nor on how
// the arena is cut into buckets, and a graph replay computes what an eager step does.
#include "common.cuh"

#define CC_MAXP 16                                                // = ROBUST_MAXP: the rows live in registers

struct CcArgs {
  const float* grad_in;                   // [slots][slot_stride] worker slots (PS memory)
  long long slot_stride;
  int n;                                  // rows the rule runs on
  const int* rows;                        // [n][T] worker slot of row i of tensor t, or null: row i is slot i
  TileView tv;
  const float* center;                    // [D] v
  double* partials;                       // [ntiles][n]
  float* weights;                         // [T][n]
  double tau;
  int tile_begin, tile_end;               // dist: tiles (tile_end == 0: to the end of the arena)
  int t_begin, t_end;                     // weights: tensors (t_end == 0: every tensor); buckets hold whole tensors
  double* dist;                           // model scope: [T][n] the per-tensor d_i, folded in tile order
  // worker buckets (appended): row i is the bucket row of wb_mask[i] / wb_scale[i] (bucketing.cu), formed in registers
  const unsigned int* wb_mask;
  const float* wb_scale;
};

__global__ void __launch_bounds__(DRC_THREADS) cc_dist_kernel(const __grid_constant__ CcArgs a) {
  __shared__ double s_part[DRC_THREADS / 32][CC_MAXP];
  const int n = a.n, T = a.tv.ntensors;
  const int tile_end = a.tile_end > 0 ? a.tile_end : a.tv.ntiles;
  for (int tile = a.tile_begin + blockIdx.x; tile < tile_end; tile += gridDim.x) {
    int tensor;
    const int valid = tile_valid(a.tv, tile, tensor);
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    const int lane_valid = valid - (int)threadIdx.x * 4;        // real elements of this thread (<= 0: padding only)
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 x[CC_MAXP];
    if (lane_valid > 0) v = *reinterpret_cast<const float4*>(a.center + idx);
#pragma unroll
    for (int i = 0; i < CC_MAXP; ++i) {
      x[i] = v;
      if (i < n && lane_valid > 0) {
        const int slot = a.rows ? a.rows[i * T + tensor] : i;
        x[i] = ld_f4(reinterpret_cast<const float4*>(a.grad_in + slot * a.slot_stride + idx));
      }
    }
#pragma unroll
    for (int i = 0; i < CC_MAXP; ++i) {
      if (i < n) {
        double d = 0.0;
        if (lane_valid > 0) {
          const double e0 = __dsub_rn((double)x[i].x, (double)v.x);
          d = __dmul_rn(e0, e0);
          if (lane_valid > 1) { const double e = __dsub_rn((double)x[i].y, (double)v.y); d = __dadd_rn(d, __dmul_rn(e, e)); }
          if (lane_valid > 2) { const double e = __dsub_rn((double)x[i].z, (double)v.z); d = __dadd_rn(d, __dmul_rn(e, e)); }
          if (lane_valid > 3) { const double e = __dsub_rn((double)x[i].w, (double)v.w); d = __dadd_rn(d, __dmul_rn(e, e)); }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) d = __dadd_rn(d, __shfl_xor_sync(0xffffffffu, d, o));
        if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5][i] = d;
      }
    }
    __syncthreads();
    if ((int)threadIdx.x < n) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < DRC_THREADS / 32; ++w) s = __dadd_rn(s, s_part[w][threadIdx.x]);
      a.partials[(long long)tile * n + threadIdx.x] = s;
    }
    __syncthreads();
  }
}

// cc_dist_kernel over the n = nb worker-bucket rows (--bucketing): row i is formed per coordinate in fp32 from its member slots
// in ascending order, starting from -0.0f, then times wb_scale[i] (aggregate_update.cu mode 7's rows, codes/oracle.py::
// wbucket_rows).  The rest is cc_dist_kernel's fixed-order reduction; a kernel of its own keeps cc_dist_kernel's machine code.
__global__ void __launch_bounds__(DRC_THREADS) cc_dist_wbucket_kernel(const __grid_constant__ CcArgs a) {
  __shared__ double s_part[DRC_THREADS / 32][CC_MAXP];
  const int n = a.n;
  const int tile_end = a.tile_end > 0 ? a.tile_end : a.tv.ntiles;
  for (int tile = a.tile_begin + blockIdx.x; tile < tile_end; tile += gridDim.x) {
    int tensor;
    const int valid = tile_valid(a.tv, tile, tensor);
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    const int lane_valid = valid - (int)threadIdx.x * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane_valid > 0) v = *reinterpret_cast<const float4*>(a.center + idx);
#pragma unroll
    for (int i = 0; i < CC_MAXP; ++i) {
      if (i < n) {
        double d = 0.0;
        if (lane_valid > 0) {
          float4 y = make_float4(-0.f, -0.f, -0.f, -0.f);
          for (unsigned int m = a.wb_mask[i]; m; m &= m - 1u) {
            const float4 x = ld_f4(reinterpret_cast<const float4*>(a.grad_in + (__ffs(m) - 1) * a.slot_stride + idx));
            y.x = __fadd_rn(y.x, x.x); y.y = __fadd_rn(y.y, x.y); y.z = __fadd_rn(y.z, x.z); y.w = __fadd_rn(y.w, x.w);
          }
          const float sc = a.wb_scale[i];
          y.x = __fmul_rn(y.x, sc); y.y = __fmul_rn(y.y, sc); y.z = __fmul_rn(y.z, sc); y.w = __fmul_rn(y.w, sc);
          const double e0 = __dsub_rn((double)y.x, (double)v.x);
          d = __dmul_rn(e0, e0);
          if (lane_valid > 1) { const double e = __dsub_rn((double)y.y, (double)v.y); d = __dadd_rn(d, __dmul_rn(e, e)); }
          if (lane_valid > 2) { const double e = __dsub_rn((double)y.z, (double)v.z); d = __dadd_rn(d, __dmul_rn(e, e)); }
          if (lane_valid > 3) { const double e = __dsub_rn((double)y.w, (double)v.w); d = __dadd_rn(d, __dmul_rn(e, e)); }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) d = __dadd_rn(d, __shfl_xor_sync(0xffffffffu, d, o));
        if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5][i] = d;
      }
    }
    __syncthreads();
    if ((int)threadIdx.x < n) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < DRC_THREADS / 32; ++w) s = __dadd_rn(s, s_part[w][threadIdx.x]);
      a.partials[(long long)tile * n + threadIdx.x] = s;
    }
    __syncthreads();
  }
}

// One warp per tensor, lane i < n folds row i's partials over the tensor's tiles in tile order, then writes its weight.  The
// loads of a batch of CC_FOLD tiles are issued together and the sum stays in order: the fold of a 2304-tile tensor is bound by
// the load latency of its batches
#define CC_FOLD 32
// cc_fold_tensor / cc_weight restate cc_weights_kernel's fold and weight for the model-scope kernels below; the per-tensor
// kernel keeps its own copy so that its machine code stays what it was
__device__ __forceinline__ double cc_fold_tensor(const CcArgs& a, int tensor, int i) {
  const int n = a.n;
  const TensorMeta m = a.tv.meta[tensor];
  const int t0 = (int)(m.offset / DRC_TILE), t1 = t0 + (int)((m.numel + DRC_TILE - 1) / DRC_TILE);
  const double* p = a.partials + i;
  double d = 0.0;
  int t = t0;
  for (; t + CC_FOLD <= t1; t += CC_FOLD) {
    double b[CC_FOLD];
#pragma unroll
    for (int k = 0; k < CC_FOLD; ++k) b[k] = p[(long long)(t + k) * n];
#pragma unroll
    for (int k = 0; k < CC_FOLD; ++k) d = __dadd_rn(d, b[k]);
  }
  for (; t < t1; ++t) d = __dadd_rn(d, p[(long long)t * n]);
  return d;
}

__device__ __forceinline__ float cc_weight(double d, double tau, int n) {
  if (!(d < INFINITY)) return 0.f;                               // NaN or +Inf: the row is never read
  if (d == 0.0) return (float)__ddiv_rn(1.0, (double)n);
  return (float)__ddiv_rn(fmin(1.0, __ddiv_rn(tau, __dsqrt_rn(d))), (double)n);
}

__global__ void __launch_bounds__(DRC_THREADS) cc_weights_kernel(const __grid_constant__ CcArgs a) {
  const int t_end = a.t_end > 0 ? a.t_end : a.tv.ntensors;
  const int tensor = a.t_begin + (int)(blockIdx.x * (DRC_THREADS / 32) + (threadIdx.x >> 5));
  const int i = threadIdx.x & 31, n = a.n;
  if (tensor >= t_end || i >= n) return;
  const TensorMeta m = a.tv.meta[tensor];
  const int t0 = (int)(m.offset / DRC_TILE), t1 = t0 + (int)((m.numel + DRC_TILE - 1) / DRC_TILE);
  const double* p = a.partials + i;
  double d = 0.0;
  int t = t0;
  for (; t + CC_FOLD <= t1; t += CC_FOLD) {
    double b[CC_FOLD];
#pragma unroll
    for (int k = 0; k < CC_FOLD; ++k) b[k] = p[(long long)(t + k) * n];
#pragma unroll
    for (int k = 0; k < CC_FOLD; ++k) d = __dadd_rn(d, b[k]);
  }
  for (; t < t1; ++t) d = __dadd_rn(d, p[(long long)t * n]);
  float w;
  if (!(d < INFINITY)) w = 0.f;                                  // NaN or +Inf: the row is never read
  else if (d == 0.0) w = (float)__ddiv_rn(1.0, (double)n);
  else w = (float)__ddiv_rn(fmin(1.0, __ddiv_rn(a.tau, __dsqrt_rn(d))), (double)n);
  a.weights[tensor * n + i] = w;
}

// Model scope (--rule-scope model), two kernels.  cc_fold_kernel: the per-tensor fold of cc_weights_kernel, in parallel over
// the tensors, into dist[T][n].  cc_model_weights_kernel: one CTA; lane i of warp 0 sums dist[t][i] over t in ascending order
// (a NaN or Inf in one tensor reaches the sum), forms w_i with cc_weight, and the CTA writes w into all T rows of weights, so
// mode 5 clips every tensor with the one whole-model norm.
__global__ void __launch_bounds__(DRC_THREADS) cc_fold_kernel(const __grid_constant__ CcArgs a) {
  const int tensor = (int)(blockIdx.x * (DRC_THREADS / 32) + (threadIdx.x >> 5));
  const int i = threadIdx.x & 31, n = a.n;
  if (tensor >= a.tv.ntensors || i >= n) return;
  a.dist[tensor * n + i] = cc_fold_tensor(a, tensor, i);
}

__global__ void __launch_bounds__(DRC_THREADS) cc_model_weights_kernel(const __grid_constant__ CcArgs a) {
  __shared__ float s_w[CC_MAXP];
  const int n = a.n, T = a.tv.ntensors;
  if ((int)threadIdx.x < n) {
    const int i = threadIdx.x;
    double d = 0.0;
    int t = 0;
    for (; t + CC_FOLD <= T; t += CC_FOLD) {
      double b[CC_FOLD];
#pragma unroll
      for (int k = 0; k < CC_FOLD; ++k) b[k] = a.dist[(t + k) * n + i];
#pragma unroll
      for (int k = 0; k < CC_FOLD; ++k) d = __dadd_rn(d, b[k]);
    }
    for (; t < T; ++t) d = __dadd_rn(d, a.dist[t * n + i]);
    s_w[i] = cc_weight(d, a.tau, n);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < T * n; k += DRC_THREADS) a.weights[k] = s_w[k % n];
}

extern "C" int drc_cc_dist(const CcArgs* args, int grid, cudaStream_t stream) {
  if (args->n < 1 || args->n > CC_MAXP || !args->center || !args->partials || grid < 1) return (int)cudaErrorInvalidValue;
  if (args->wb_mask) {                                           // worker-bucket rows: no row table
    if (!args->wb_scale || args->rows) return (int)cudaErrorInvalidValue;
    cc_dist_wbucket_kernel<<<grid, DRC_THREADS, 0, stream>>>(*args);
    return (int)cudaGetLastError();
  }
  cc_dist_kernel<<<grid, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_cc_weights(const CcArgs* args, cudaStream_t stream) {
  if (args->n < 1 || args->n > CC_MAXP || !args->partials || !args->weights || !(args->tau > 0.0 && args->tau < INFINITY))
    return (int)cudaErrorInvalidValue;
  const int t_end = args->t_end > 0 ? args->t_end : args->tv.ntensors;
  if (args->t_begin < 0 || t_end <= args->t_begin || t_end > args->tv.ntensors) return (int)cudaErrorInvalidValue;
  const int warps = DRC_THREADS / 32;
  cc_weights_kernel<<<(t_end - args->t_begin + warps - 1) / warps, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_cc_model_weights(const CcArgs* args, cudaStream_t stream) {
  if (args->n < 1 || args->n > CC_MAXP || !args->partials || !args->weights || !args->dist ||
      !(args->tau > 0.0 && args->tau < INFINITY) || args->tv.ntensors < 1)
    return (int)cudaErrorInvalidValue;
  const int warps = DRC_THREADS / 32;
  cc_fold_kernel<<<(args->tv.ntensors + warps - 1) / warps, DRC_THREADS, 0, stream>>>(*args);
  cc_model_weights_kernel<<<1, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
// cc_fold_kernel alone: ARC's whole-model norm (arc.cu) folds its per-tile partials [ntiles][n] into dist[T][n] with it
extern "C" int drc_cc_fold(const CcArgs* args, cudaStream_t stream) {
  if (args->n < 1 || args->n > CC_MAXP || !args->partials || !args->dist || args->tv.ntensors < 1)
    return (int)cudaErrorInvalidValue;
  const int warps = DRC_THREADS / 32;
  cc_fold_kernel<<<(args->tv.ntensors + warps - 1) / warps, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_sizeof_CcArgs() { return (int)sizeof(CcArgs); }
