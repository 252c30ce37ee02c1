// The mimic attack (Karimireddy, He and Jaggi, ICLR 2022), applied by the PS to the liar slots of the grad_in slab
// (codes/adversary.py ``mimic_step`` is the fp64 oracle).  Every liar slot becomes a bit copy of the honest slot k with the
// largest <x_i, z> over the whole model, z a unit direction the PS learns during the job's first W steps (t = step - 1 < W):
//
//   m' = fp32((t m + c) / (t + 1))          c the fp64 honest mean, m the running mean of the honest means
//   w_i = s_i - <m', z>                      s_i = <x_i, z>, both whole-model fp64 sums (= <x_i - m', z> up to rounding)
//   u = t z + sum_i w_i (x_i - m')           fp64, honest slots in ascending order
//   z = fp32(u / ||u||)                      unchanged when ||u|| = 0
//
// One launch per step after the last gradient bucket (the target needs whole-model sums), six kernels:
//   mimic_dot_kernel     per tile: s_i (and, in warm-up, m' and <m', z>) as fp64 per-tile partials
//   mimic_fold_kernel    one CTA per tensor: the partials folded in tile order
//   mimic_select_kernel  one CTA: the tensors summed in ascending order, the target k (NaN largest, ties to the lower slot), w_i
//   mimic_write_kernel   per tile: x_k into every liar slot; in warm-up u and the per-tile partials of ||u||^2
//   mimic_fold_kernel    (warm-up) ||u||^2 per tensor
//   mimic_scale_kernel   (warm-up) z = fp32(u / ||u||)
// The warm-up kernels are launched every step and return on the device after step W, so one captured graph serves the whole
// job.  No floating-point atomics: results do not depend on the grid size.  Padding is never read into a sum and never written.
#include "common.cuh"

#define MIMIC_MAXP 16                    // = ROBUST_MAXP
#define MIMIC_NQ(P) ((P) + 1)            // partials per tile: s_i, then <m', z>

struct MimicArgs {
  float* grad_in;                        // [P][slot_stride] worker slots (PS memory)
  long long slot_stride;
  int P;
  int warmup;                            // W: the state is updated while step - 1 < W
  TileView tv;
  const unsigned int* adv_bitmap;        // [adv_len] liar bitmap per step (bit w = slot w lies)
  int adv_len;
  const unsigned long long* step_ptr;
  float* m;                              // [slot_stride] running mean of the honest means (state)
  float* z;                              // [slot_stride] unit direction (state)
  double* u;                             // [slot_stride] warm-up scratch: the unnormalised direction
  double* partials;                      // [ntiles][MIMIC_NQ(P)]
  double* fold;                          // [ntensors][MIMIC_NQ(P)]
  double* upart;                         // [ntiles] ||u||^2 per tile
  double* ufold;                         // [ntensors] ||u||^2 per tensor
  double* w;                             // [P] w_i of the honest slots (0 for the liars)
  int* target;                           // [1] the slot the liars copy
};

struct MimicStep {
  unsigned int liars, honest;
  unsigned long long t;                  // warm-up index: step - 1
  bool warm;
};

__device__ __forceinline__ MimicStep mimic_step_of(const MimicArgs& a) {
  MimicStep s;
  const unsigned long long step = *a.step_ptr;
  const unsigned int all = (1u << a.P) - 1u;
  s.liars = a.adv_len > 0 ? a.adv_bitmap[step % (unsigned long long)a.adv_len] & all : 0u;
  s.honest = ~s.liars & all;
  s.t = step - 1ull;
  s.warm = s.t < (unsigned long long)a.warmup;
  return s;
}

__device__ __forceinline__ float lane4(const float4& v, int k) { return k == 0 ? v.x : k == 1 ? v.y : k == 2 ? v.z : v.w; }

// a float4 with the lanes at and past lane_valid set to 0 (padding takes no part in a sum)
__device__ __forceinline__ float4 load_valid(const float* p, int lane_valid) {
  float4 v = ld_f4(reinterpret_cast<const float4*>(p));
  if (lane_valid < 4) {
    if (lane_valid < 2) v.y = 0.f;
    if (lane_valid < 3) v.z = 0.f;
    v.w = 0.f;
  }
  return v;
}

// x summed over the CTA into s_part[warp][q] (warp shuffles in a fixed pattern; the warps are folded later, in order)
__device__ __forceinline__ void mimic_warp_partial(double x, double* s_part, int q) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  if ((threadIdx.x & 31) == 0) s_part[(threadIdx.x >> 5) * MIMIC_NQ(MIMIC_MAXP) + q] = x;
}

__global__ void __launch_bounds__(DRC_THREADS) mimic_dot_kernel(const __grid_constant__ MimicArgs a) {
  __shared__ double s_part[(DRC_THREADS / 32) * MIMIC_NQ(MIMIC_MAXP)];
  const MimicStep st = mimic_step_of(a);
  if (st.honest == 0u) return;
  const int P = a.P, Q = MIMIC_NQ(a.P);
  const double nh = (double)__popc(st.honest), t = (double)st.t;
  for (int tile = blockIdx.x; tile < a.tv.ntiles; tile += gridDim.x) {
    int tensor;
    const int valid = tile_valid(a.tv, tile, tensor);
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    const int lane_valid = valid - (int)threadIdx.x * 4;
    const float4 z = lane_valid > 0 ? load_valid(a.z + idx, lane_valid) : make_float4(0.f, 0.f, 0.f, 0.f);
    double c[4] = {0.0, 0.0, 0.0, 0.0};
    for (int i = 0; i < P; ++i) {
      if ((st.honest >> i) & 1u) {
        const float4 x = lane_valid > 0 ? load_valid(a.grad_in + i * a.slot_stride + idx, lane_valid)
                                        : make_float4(0.f, 0.f, 0.f, 0.f);
        double d = 0.0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          d = fma((double)lane4(x, k), (double)lane4(z, k), d);
          c[k] = __dadd_rn(c[k], (double)lane4(x, k));
        }
        mimic_warp_partial(d, s_part, i);
      } else if ((threadIdx.x & 31) == 0) {
        s_part[(threadIdx.x >> 5) * MIMIC_NQ(MIMIC_MAXP) + i] = 0.0;
      }
    }
    if (st.warm) {                                             // m' = fp32((t m + c) / (t + 1)), written back into m
      double d = 0.0;
      if (lane_valid > 0) {
        const float4 m = *reinterpret_cast<const float4*>(a.m + idx);
        float r[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          r[k] = (float)(__dadd_rn(__dmul_rn(t, (double)lane4(m, k)), c[k] / nh) / (t + 1.0));
          if (k < lane_valid) d = fma((double)r[k], (double)lane4(z, k), d);
        }
        if (lane_valid >= 4) {
          *reinterpret_cast<float4*>(a.m + idx) = make_float4(r[0], r[1], r[2], r[3]);
        } else {
          a.m[idx] = r[0];
          if (lane_valid > 1) a.m[idx + 1] = r[1];
          if (lane_valid > 2) a.m[idx + 2] = r[2];
        }
      }
      mimic_warp_partial(d, s_part, P);
    } else if ((threadIdx.x & 31) == 0) {
      s_part[(threadIdx.x >> 5) * MIMIC_NQ(MIMIC_MAXP) + P] = 0.0;
    }
    __syncthreads();
    for (int q = threadIdx.x; q < Q; q += DRC_THREADS) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < DRC_THREADS / 32; ++w) s += s_part[w * MIMIC_NQ(MIMIC_MAXP) + q];
      a.partials[(long long)tile * Q + q] = s;
    }
    __syncthreads();
  }
}

// One CTA per tensor: its per-tile partials folded in tile order.  norm = 0: the Q dot partials into fold; norm = 1 (warm-up
// only): ||u||^2 into ufold
__global__ void __launch_bounds__(DRC_THREADS) mimic_fold_kernel(const __grid_constant__ MimicArgs a, int norm) {
  const MimicStep st = mimic_step_of(a);
  if (st.honest == 0u || (norm && !st.warm)) return;
  const TensorMeta m = a.tv.meta[blockIdx.x];
  const int t0 = (int)(m.offset / DRC_TILE), t1 = t0 + (int)((m.numel + DRC_TILE - 1) / DRC_TILE);
  const int Q = norm ? 1 : MIMIC_NQ(a.P);
  const double* src = norm ? a.upart : a.partials;
  double* dst = norm ? a.ufold : a.fold;
  for (int q = threadIdx.x; q < Q; q += DRC_THREADS) {
    double s = 0.0;
    for (int t = t0; t < t1; ++t) s += src[(long long)t * Q + q];
    dst[(long long)blockIdx.x * Q + q] = s;
  }
}

// One CTA: s_i and <m', z> summed over the tensors in ascending order, then the target (np.argmax over the honest slots in
// ascending order: the first NaN, else the first largest) and w_i = s_i - <m', z>
__global__ void __launch_bounds__(DRC_THREADS) mimic_select_kernel(const __grid_constant__ MimicArgs a) {
  __shared__ double s_sum[MIMIC_NQ(MIMIC_MAXP)];
  const MimicStep st = mimic_step_of(a);
  if (st.honest == 0u) return;
  const int P = a.P, Q = MIMIC_NQ(a.P), T = a.tv.ntensors;
  for (int q = threadIdx.x; q < Q; q += DRC_THREADS) {
    double s = 0.0;
    for (int t = 0; t < T; ++t) s += a.fold[(long long)t * Q + q];
    s_sum[q] = s;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  int k = -1;
  for (int i = 0; i < P; ++i) {
    if (!((st.honest >> i) & 1u)) continue;
    const double si = s_sum[i];
    if (k < 0 || (s_sum[k] == s_sum[k] && (si != si || si > s_sum[k]))) k = i;
  }
  *a.target = k;
  for (int i = 0; i < P; ++i) a.w[i] = ((st.honest >> i) & 1u) ? __dsub_rn(s_sum[i], s_sum[P]) : 0.0;
}

__global__ void __launch_bounds__(DRC_THREADS) mimic_write_kernel(const __grid_constant__ MimicArgs a) {
  __shared__ double s_part[DRC_THREADS / 32];
  const MimicStep st = mimic_step_of(a);
  if (st.honest == 0u) return;
  const int P = a.P, k = *a.target;
  const double t = (double)st.t;
  for (int tile = blockIdx.x; tile < a.tv.ntiles; tile += gridDim.x) {
    int tensor;
    const int valid = tile_valid(a.tv, tile, tensor);
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    const int lane_valid = valid - (int)threadIdx.x * 4;
    if (st.liars != 0u && lane_valid > 0) {                    // the liars' copy of x_k, bit for bit
      const float4 xk = ld_f4(reinterpret_cast<const float4*>(a.grad_in + k * a.slot_stride + idx));
      for (int w = 0; w < P; ++w) {
        if (!((st.liars >> w) & 1u)) continue;
        float* p = a.grad_in + w * a.slot_stride + idx;
        if (lane_valid >= 4) {
          st_f4(reinterpret_cast<float4*>(p), xk);
        } else {
          p[0] = xk.x;
          if (lane_valid > 1) p[1] = xk.y;
          if (lane_valid > 2) p[2] = xk.z;
        }
      }
    }
    if (!st.warm) continue;
    // u = t z + sum_i w_i (x_i - m'), fp64 without contraction (the oracle's order), and this tile's share of ||u||^2
    double n2 = 0.0;
    if (lane_valid > 0) {
      const float4 z = load_valid(a.z + idx, lane_valid), m = load_valid(a.m + idx, lane_valid);
      double u[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) u[q] = __dmul_rn(t, (double)lane4(z, q));
      for (int i = 0; i < P; ++i) {
        if (!((st.honest >> i) & 1u)) continue;
        const double wi = a.w[i];
        const float4 x = load_valid(a.grad_in + i * a.slot_stride + idx, lane_valid);
#pragma unroll
        for (int q = 0; q < 4; ++q) u[q] = __dadd_rn(u[q], __dmul_rn(wi, __dsub_rn((double)lane4(x, q), (double)lane4(m, q))));
      }
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (q < lane_valid) {
          a.u[idx + q] = u[q];
          n2 = fma(u[q], u[q], n2);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n2 += __shfl_xor_sync(0xffffffffu, n2, o);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = n2;
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < DRC_THREADS / 32; ++w) s += s_part[w];
      a.upart[tile] = s;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(DRC_THREADS) mimic_scale_kernel(const __grid_constant__ MimicArgs a) {
  __shared__ double s_norm;
  const MimicStep st = mimic_step_of(a);
  if (st.honest == 0u || !st.warm) return;
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int t = 0; t < a.tv.ntensors; ++t) s += a.ufold[t];
    s_norm = sqrt(s);
  }
  __syncthreads();
  const double nrm = s_norm;
  if (nrm == 0.0) return;                                      // z unchanged
  for (int tile = blockIdx.x; tile < a.tv.ntiles; tile += gridDim.x) {
    int tensor;
    const int valid = tile_valid(a.tv, tile, tensor);
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    const int lane_valid = valid - (int)threadIdx.x * 4;
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (q < lane_valid) a.z[idx + q] = (float)(a.u[idx + q] / nrm);
  }
}

extern "C" int drc_mimic_step(const MimicArgs* a, int grid, cudaStream_t stream) {
  if (a->P < 1 || a->P > MIMIC_MAXP || a->warmup < 0 || grid < 1 || a->tv.ntensors < 1 || !a->m || !a->z || !a->u ||
      !a->partials || !a->fold || !a->upart || !a->ufold || !a->w || !a->target)
    return (int)cudaErrorInvalidValue;
  const int T = a->tv.ntensors;
  mimic_dot_kernel<<<grid, DRC_THREADS, 0, stream>>>(*a);
  mimic_fold_kernel<<<T, DRC_THREADS, 0, stream>>>(*a, 0);
  mimic_select_kernel<<<1, DRC_THREADS, 0, stream>>>(*a);
  mimic_write_kernel<<<grid, DRC_THREADS, 0, stream>>>(*a);
  mimic_fold_kernel<<<T, DRC_THREADS, 0, stream>>>(*a, 1);
  mimic_scale_kernel<<<grid, DRC_THREADS, 0, stream>>>(*a);
  return (int)cudaGetLastError();
}
extern "C" int drc_sizeof_MimicArgs() { return (int)sizeof(MimicArgs); }
