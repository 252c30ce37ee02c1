// C12: the ALIE and min-max attacks, applied by the PS to the liar slots of the grad_in slab (codes/adversary.py holds the
// fp64 oracle of both).  The liar set is the step's bitmap adv_bitmap[step % adv_len], read on the device, so the attack
// runs inside the captured graph.  Workers push their true gradient; every liar slot is then overwritten with one row
// built from the per-coordinate mean mu and population standard deviation sigma of the honest slots of each tensor:
//
//   ALIE    (Baruch et al., NeurIPS 2019):         mu - z * sigma                       one pass: attack_stats_kernel
//   min-max (Shejwalkar & Houmansadr, NDSS 2021):  mu - gamma * sigma, with the largest gamma such that no honest row is
//            farther from it than the largest honest pairwise distance Dmax (per tensor; closed form, see attack_solve_kernel)
//            three kernels: stats (mu, sigma + per-tile fp64 partials) -> solve (one CTA per tensor) -> write
//   IPM     (Xie, Koyejo and Gupta, UAI 2019):     -eps * mu                            one pass: attack_ipm_kernel
// (mimic, which copies one honest slot, is in mimic.cu)
//
// Determinism: every per-coordinate statistic is a fixed-order fp64 sum over the honest rows in slot order, with the
// roundings of the oracle (no contracted multiply-adds), so an ALIE row is the oracle's fp64 row rounded to fp32; the per-tensor
// sums of min-max are per-tile partials (warp shuffles, then the 8 warps in order) folded in tile order by the solve.  No
// floating-point atomics: results do not depend on the grid size or on how the arena is cut into buckets.
#include "common.cuh"

#define ATTACK_MAXP 16                                            // = ROBUST_MAXP: the rows live in registers
#define ATTACK_NQ(P) (2 * (P) + 1 + (P) * ((P) - 1) / 2)          // partials per tile: a_i, b_i, c, pair distances
#define ATTACK_MAXQ ATTACK_NQ(ATTACK_MAXP)
#define ATTACK_ALIE 5                                             // ATTACK_* codes of codes/adversary.py
#define ATTACK_MINMAX 6
#define ATTACK_IPM 7

struct AttackArgs {
  float* grad_in;                         // [P][slot_stride] worker slots (PS memory)
  long long slot_stride;
  int P;
  int mode;                               // ATTACK_ALIE | ATTACK_MINMAX | ATTACK_IPM
  TileView tv;
  const unsigned int* adv_bitmap;         // [adv_len] liar bitmap per step (bit w = slot w lies)
  int adv_len;
  const unsigned long long* step_ptr;
  double z;                               // ALIE's z; IPM's eps
  float* stats;                           // min-max: [2][slot_stride] mu, sigma (fp32)
  double* partials;                       // min-max: [ntiles][ATTACK_NQ(P)]
  double* gamma;                          // min-max: [ntensors]
  int tile_begin, tile_end;               // stats / write: tiles (tile_end == 0: to the end of the arena)
  int t_begin, t_end;                     // solve: tensors (t_end == 0: every tensor); buckets hold whole tensors
  double* fold;                           // model scope: [ntensors][ATTACK_NQ(P)] the partials folded per tensor
};

__device__ __forceinline__ unsigned int liar_mask(const AttackArgs& a) {
  if (a.adv_len <= 0) return 0u;
  const unsigned long long step = *a.step_ptr;
  return a.adv_bitmap[step % (unsigned long long)a.adv_len] & ((1u << a.P) - 1u);
}

__device__ __forceinline__ float lane_of(const float4& v, int k) { return k == 0 ? v.x : k == 1 ? v.y : k == 2 ? v.z : v.w; }

// x summed over the CTA into s_part[warp][q] (warp shuffles in a fixed pattern; the warps are folded later, in order)
__device__ __forceinline__ void warp_partial(double x, double* s_part, int q) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  if ((threadIdx.x & 31) == 0) s_part[(threadIdx.x >> 5) * ATTACK_MAXQ + q] = x;
}

__global__ void __launch_bounds__(DRC_THREADS) attack_stats_kernel(const __grid_constant__ AttackArgs a) {
  __shared__ double s_part[(DRC_THREADS / 32) * ATTACK_MAXQ];
  const unsigned int liars = liar_mask(a);
  const unsigned int honest = ~liars & ((1u << a.P) - 1u);
  if (liars == 0u || honest == 0u) return;
  const double nh = (double)__popc(honest);
  const int P = a.P, Q = ATTACK_NQ(a.P);
  const int tile_end = a.tile_end > 0 ? a.tile_end : a.tv.ntiles;
  for (int tile = a.tile_begin + blockIdx.x; tile < tile_end; tile += gridDim.x) {
    int tensor;
    const int valid = tile_valid(a.tv, tile, tensor);
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    const int lane_valid = valid - (int)threadIdx.x * 4;        // real elements of this thread (<= 0: padding only)
    float4 v[ATTACK_MAXP];
#pragma unroll
    for (int i = 0; i < ATTACK_MAXP; ++i) {
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (i < P && ((honest >> i) & 1u) && lane_valid > 0) {
        v[i] = ld_f4(reinterpret_cast<const float4*>(a.grad_in + i * a.slot_stride + idx));
        if (lane_valid < 4) {                                   // padding lanes take no part
          if (lane_valid < 2) v[i].y = 0.f;
          if (lane_valid < 3) v[i].z = 0.f;
          v[i].w = 0.f;
        }
      }
    }
    double mu[4] = {0.0, 0.0, 0.0, 0.0}, sd[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
    for (int i = 0; i < ATTACK_MAXP; ++i)
      if (i < P && ((honest >> i) & 1u)) {
#pragma unroll
        for (int k = 0; k < 4; ++k) mu[k] += (double)lane_of(v[i], k);
      }
#pragma unroll
    for (int k = 0; k < 4; ++k) mu[k] = mu[k] / nh;
#pragma unroll
    for (int i = 0; i < ATTACK_MAXP; ++i)
      if (i < P && ((honest >> i) & 1u)) {
#pragma unroll
        for (int k = 0; k < 4; ++k) { const double d = (double)lane_of(v[i], k) - mu[k]; sd[k] = __dadd_rn(sd[k], __dmul_rn(d, d)); }
      }
#pragma unroll
    for (int k = 0; k < 4; ++k) sd[k] = sqrt(sd[k] / nh);

    if (a.mode == ATTACK_ALIE) {                                // the liars' row, straight from the registers
      if (lane_valid > 0) {
        float r[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) r[k] = (float)__dsub_rn(mu[k], __dmul_rn(a.z, sd[k]));
        for (int w = 0; w < P; ++w)
          if ((liars >> w) & 1u) store_row(a.grad_in + w * a.slot_stride + idx, r, lane_valid);
      }
      continue;
    }
    // min-max: mu and sigma for the write pass, then this tile's share of a_i, b_i, c and the honest pair distances
    if (lane_valid > 0) {
      *reinterpret_cast<float4*>(a.stats + idx) = make_float4((float)mu[0], (float)mu[1], (float)mu[2], (float)mu[3]);
      *reinterpret_cast<float4*>(a.stats + a.slot_stride + idx) = make_float4((float)sd[0], (float)sd[1], (float)sd[2], (float)sd[3]);
    }
#pragma unroll
    for (int i = 0; i < ATTACK_MAXP; ++i) {
      if (i < P) {
        if ((honest >> i) & 1u) {
          double ai = 0.0, bi = 0.0;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const double e = mu[k] - (double)lane_of(v[i], k);   // mu - g_i
            ai = fma(e, e, ai);
            bi = fma(-e, sd[k], bi);                             // <mu - g_i, p>, p = -sigma
          }
          warp_partial(ai, s_part, i);
          warp_partial(bi, s_part, P + i);
        } else if ((threadIdx.x & 31) == 0) {
          s_part[(threadIdx.x >> 5) * ATTACK_MAXQ + i] = 0.0;
          s_part[(threadIdx.x >> 5) * ATTACK_MAXQ + P + i] = 0.0;
        }
      }
    }
    warp_partial(sd[0] * sd[0] + sd[1] * sd[1] + sd[2] * sd[2] + sd[3] * sd[3], s_part, 2 * P);
#pragma unroll
    for (int j = 1; j < ATTACK_MAXP; ++j) {
#pragma unroll
      for (int i = 0; i < j; ++i) {
        if (j < P) {
          const int q = 2 * P + 1 + j * (j - 1) / 2 + i;
          if (((honest >> i) & 1u) && ((honest >> j) & 1u)) {
            double d = 0.0;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const double e = (double)lane_of(v[i], k) - (double)lane_of(v[j], k);
              d = fma(e, e, d);
            }
            warp_partial(d, s_part, q);
          } else if ((threadIdx.x & 31) == 0) {
            s_part[(threadIdx.x >> 5) * ATTACK_MAXQ + q] = 0.0;
          }
        }
      }
    }
    __syncthreads();
    for (int q = threadIdx.x; q < Q; q += DRC_THREADS) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < DRC_THREADS / 32; ++w) s += s_part[w * ATTACK_MAXQ + q];
      a.partials[(long long)tile * Q + q] = s;
    }
    __syncthreads();
  }
}

// max / min that return NaN as soon as one operand is NaN (np.max / np.min do): a NaN in the honest rows poisons gamma
__device__ __forceinline__ double max_nan(double x, double y) { return (x != x || x > y) ? x : y; }
__device__ __forceinline__ double min_nan(double x, double y) { return (x != x || x < y) ? x : y; }

// gamma from the folded sums s_sum[ATTACK_NQ(P)] (a_i, b_i, c, pair distances) of the honest rows:
//   Dmax^2 = max_{i<j in H} ||g_i - g_j||^2,  c = ||p||^2,
//   gamma  = min_{i in H} largest root of  c g^2 + 2 b_i g + (a_i - Dmax^2) = 0   (||mu + g p - g_i||^2 = Dmax^2)
// Both roots' forms are the same number; the one without cancellation is used (b_i > 0: (Dmax^2 - a_i) / (b_i + sqrt(disc))).
__device__ __forceinline__ double minmax_solve(const double* s_sum, int P, unsigned int honest) {
  double D2 = 0.0;
  for (int j = 1; j < P; ++j)
    for (int i = 0; i < j; ++i)
      if (((honest >> i) & 1u) && ((honest >> j) & 1u)) D2 = max_nan(s_sum[2 * P + 1 + j * (j - 1) / 2 + i], D2);
  const double c = s_sum[2 * P];
  double gamma;
  if (c == 0.0) {
    gamma = 0.0;                                               // every honest row equal: the liars send them too
  } else {
    gamma = INFINITY;
    for (int i = 0; i < P; ++i) {
      if (!((honest >> i) & 1u)) continue;
      const double ai = s_sum[i], bi = s_sum[P + i];
      double disc = bi * bi + c * (D2 - ai);
      if (disc < 0.0) disc = 0.0;                              // a_i <= Dmax^2 up to rounding
      const double r = sqrt(disc);
      double g = bi <= 0.0 ? (r - bi) / c : (D2 - ai) / (bi + r);
      if (g < 0.0) g = 0.0;
      gamma = min_nan(g, gamma);                               // a NaN in Dmax^2, a_i or b_i reaches gamma through disc
    }
  }
  return gamma;
}

// One CTA per tensor: fold the tensor's per-tile partials in tile order, then solve as minmax_solve does (the kernel keeps its
// own copy of the solve so that its machine code stays what it was)
__global__ void __launch_bounds__(DRC_THREADS) attack_solve_kernel(const __grid_constant__ AttackArgs a) {
  __shared__ double s_sum[ATTACK_MAXQ];
  const unsigned int liars = liar_mask(a);
  const unsigned int honest = ~liars & ((1u << a.P) - 1u);
  if (liars == 0u || honest == 0u) return;
  const int tensor = a.t_begin + blockIdx.x;
  const TensorMeta m = a.tv.meta[tensor];
  const int t0 = (int)(m.offset / DRC_TILE), t1 = t0 + (int)((m.numel + DRC_TILE - 1) / DRC_TILE);
  const int P = a.P, Q = ATTACK_NQ(a.P);
  for (int q = threadIdx.x; q < Q; q += DRC_THREADS) {
    double s = 0.0;
    for (int t = t0; t < t1; ++t) s += a.partials[(long long)t * Q + q];
    s_sum[q] = s;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double D2 = 0.0;
  for (int j = 1; j < P; ++j)
    for (int i = 0; i < j; ++i)
      if (((honest >> i) & 1u) && ((honest >> j) & 1u)) D2 = max_nan(s_sum[2 * P + 1 + j * (j - 1) / 2 + i], D2);
  const double c = s_sum[2 * P];
  double gamma;
  if (c == 0.0) {
    gamma = 0.0;                                               // every honest row equal: the liars send them too
  } else {
    gamma = INFINITY;
    for (int i = 0; i < P; ++i) {
      if (!((honest >> i) & 1u)) continue;
      const double ai = s_sum[i], bi = s_sum[P + i];
      double disc = bi * bi + c * (D2 - ai);
      if (disc < 0.0) disc = 0.0;                              // a_i <= Dmax^2 up to rounding
      const double r = sqrt(disc);
      double g = bi <= 0.0 ? (r - bi) / c : (D2 - ai) / (bi + r);
      if (g < 0.0) g = 0.0;
      gamma = min_nan(g, gamma);                               // a NaN in Dmax^2, a_i or b_i reaches gamma through disc
    }
  }
  a.gamma[tensor] = gamma;
}

// Model scope (--attack-scope model): one gamma and one Dmax over the whole model.  attack_fold_kernel folds each tensor's
// partials in tile order as attack_solve_kernel does (one CTA per tensor) into fold[T][Q]; attack_solve_model_kernel (one CTA)
// sums every entry over the tensors in ascending order, solves once and writes gamma into every tensor.
__global__ void __launch_bounds__(DRC_THREADS) attack_fold_kernel(const __grid_constant__ AttackArgs a) {
  const unsigned int liars = liar_mask(a);
  const unsigned int honest = ~liars & ((1u << a.P) - 1u);
  if (liars == 0u || honest == 0u) return;
  const int tensor = blockIdx.x;
  const TensorMeta m = a.tv.meta[tensor];
  const int t0 = (int)(m.offset / DRC_TILE), t1 = t0 + (int)((m.numel + DRC_TILE - 1) / DRC_TILE);
  const int Q = ATTACK_NQ(a.P);
  for (int q = threadIdx.x; q < Q; q += DRC_THREADS) {
    double s = 0.0;
    for (int t = t0; t < t1; ++t) s += a.partials[(long long)t * Q + q];
    a.fold[(long long)tensor * Q + q] = s;
  }
}

__global__ void __launch_bounds__(DRC_THREADS) attack_solve_model_kernel(const __grid_constant__ AttackArgs a) {
  __shared__ double s_sum[ATTACK_MAXQ];
  __shared__ double s_gamma;
  const unsigned int liars = liar_mask(a);
  const unsigned int honest = ~liars & ((1u << a.P) - 1u);
  if (liars == 0u || honest == 0u) return;
  const int T = a.tv.ntensors, Q = ATTACK_NQ(a.P);
  for (int q = threadIdx.x; q < Q; q += DRC_THREADS) {
    double s = 0.0;
    for (int t = 0; t < T; ++t) s += a.fold[(long long)t * Q + q];
    s_sum[q] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) s_gamma = minmax_solve(s_sum, a.P, honest);
  __syncthreads();
  for (int t = threadIdx.x; t < T; t += DRC_THREADS) a.gamma[t] = s_gamma;
}

__global__ void __launch_bounds__(DRC_THREADS) attack_write_kernel(const __grid_constant__ AttackArgs a) {
  const unsigned int liars = liar_mask(a);
  const unsigned int honest = ~liars & ((1u << a.P) - 1u);
  if (liars == 0u || honest == 0u) return;
  const int tile_end = a.tile_end > 0 ? a.tile_end : a.tv.ntiles;
  for (int tile = a.tile_begin + blockIdx.x; tile < tile_end; tile += gridDim.x) {
    int tensor;
    const int valid = tile_valid(a.tv, tile, tensor);
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    const int lane_valid = valid - (int)threadIdx.x * 4;
    if (lane_valid <= 0) continue;
    const double gamma = a.gamma[tensor];
    const float4 mu = *reinterpret_cast<const float4*>(a.stats + idx);
    const float4 sd = *reinterpret_cast<const float4*>(a.stats + a.slot_stride + idx);
    float r[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) r[k] = (float)__dsub_rn((double)lane_of(mu, k), __dmul_rn(gamma, (double)lane_of(sd, k)));
    for (int w = 0; w < a.P; ++w)
      if ((liars >> w) & 1u) store_row(a.grad_in + w * a.slot_stride + idx, r, lane_valid);
  }
}

// IPM, inner-product manipulation (Xie, Koyejo and Gupta, UAI 2019): every liar sends fp32(-eps * mu), mu the honest mean of
// ALIE's kernel (the same fp64 sum in slot order, one rounded division); a.z holds eps.  Coordinate-wise, so it runs per
// gradient bucket like ALIE.  Its own kernel, so that attack_stats_kernel's machine code stays what it was.
__global__ void __launch_bounds__(DRC_THREADS) attack_ipm_kernel(const __grid_constant__ AttackArgs a) {
  const unsigned int liars = liar_mask(a);
  const unsigned int honest = ~liars & ((1u << a.P) - 1u);
  if (liars == 0u || honest == 0u) return;
  const double nh = (double)__popc(honest);
  const int tile_end = a.tile_end > 0 ? a.tile_end : a.tv.ntiles;
  for (int tile = a.tile_begin + blockIdx.x; tile < tile_end; tile += gridDim.x) {
    int tensor;
    const int valid = tile_valid(a.tv, tile, tensor);
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    const int lane_valid = valid - (int)threadIdx.x * 4;
    if (lane_valid <= 0) continue;
    double mu[4] = {0.0, 0.0, 0.0, 0.0};
    for (int i = 0; i < a.P; ++i)
      if ((honest >> i) & 1u) {
        const float4 v = ld_f4(reinterpret_cast<const float4*>(a.grad_in + i * a.slot_stride + idx));
#pragma unroll
        for (int k = 0; k < 4; ++k) mu[k] += (double)lane_of(v, k);       // padding lanes are summed but never stored
      }
    float r[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) r[k] = (float)__dmul_rn(-a.z, mu[k] / nh);
    for (int w = 0; w < a.P; ++w)
      if ((liars >> w) & 1u) store_row(a.grad_in + w * a.slot_stride + idx, r, lane_valid);
  }
}

static bool attack_args_ok(const AttackArgs* a) {
  if (a->P < 1 || a->P > ATTACK_MAXP) return false;
  if (a->mode != ATTACK_ALIE && a->mode != ATTACK_MINMAX && a->mode != ATTACK_IPM) return false;
  if (a->mode == ATTACK_MINMAX && (!a->stats || !a->partials || !a->gamma)) return false;
  return true;
}

extern "C" int drc_attack_ipm(const AttackArgs* args, int grid, cudaStream_t stream) {
  if (!attack_args_ok(args) || args->mode != ATTACK_IPM || grid < 1) return (int)cudaErrorInvalidValue;
  attack_ipm_kernel<<<grid, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_attack_stats(const AttackArgs* args, int grid, cudaStream_t stream) {
  if (!attack_args_ok(args) || args->mode == ATTACK_IPM || grid < 1) return (int)cudaErrorInvalidValue;
  attack_stats_kernel<<<grid, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_attack_solve(const AttackArgs* args, cudaStream_t stream) {
  if (!attack_args_ok(args) || args->mode != ATTACK_MINMAX) return (int)cudaErrorInvalidValue;
  const int t_end = args->t_end > 0 ? args->t_end : args->tv.ntensors;
  if (t_end <= args->t_begin) return (int)cudaErrorInvalidValue;
  attack_solve_kernel<<<t_end - args->t_begin, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_attack_solve_model(const AttackArgs* args, cudaStream_t stream) {
  if (!attack_args_ok(args) || args->mode != ATTACK_MINMAX || !args->fold || args->tv.ntensors < 1)
    return (int)cudaErrorInvalidValue;
  attack_fold_kernel<<<args->tv.ntensors, DRC_THREADS, 0, stream>>>(*args);
  attack_solve_model_kernel<<<1, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_attack_write(const AttackArgs* args, int grid, cudaStream_t stream) {
  if (!attack_args_ok(args) || args->mode != ATTACK_MINMAX || grid < 1) return (int)cudaErrorInvalidValue;
  attack_write_kernel<<<grid, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_sizeof_AttackArgs() { return (int)sizeof(AttackArgs); }
