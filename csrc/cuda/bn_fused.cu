// K10 (normalisation part): fused training-mode BatchNorm + residual add + ReLU for NHWC bf16 activations (third iteration).
//
// Design (a plain statistics + apply implementation costs four launches per layer, each far from HBM bandwidth):
//   * the forward statistics normally come out of the producing convolution's epilogue (conv_epilogue.cuh), so a layer's
//     forward is ONE streaming kernel: bn_apply_kernel (x, mean, invstd, residual -> y, ReLU fused).  bn_stats_kernel remains
//     for producers that are not ours (GEMM-served 1x1 convolutions, library fallbacks);
//   * every access is 16 bytes (8 channels per thread), 4 independent rows in flight per thread, 512-thread CTAs with up to
//     four resident per SM, and the grid is sized from the tensor (one CTA per 32 KB up to 4 per SM): the 2-4 MB late-stage
//     tensors spread over 64-128 CTAs instead of 16-32, the 16.8 MB ones keep ~64 KB of loads in flight per SM;
//   * reductions: per-thread fp32 accumulators -> fixed-order shared-memory fold -> per-CTA partial [2][C] -> the last CTA
//     (atomic ticket) folds the partials with 16-byte loads in a fixed order.  No cooperative launch, no grid barrier, no
//     cluster: safe next to any other kernel on any number of concurrent streams, and bit-deterministic (replicas of a batch
//     on different GPUs must agree exactly for the majority vote, reference: src/master/rep_master.py:162).
//
// backward: bn_bwd_reduce_kernel (dy, mask, x -> dgamma, dbeta, means)    bn_bwd_apply_kernel (dy, mask, x -> dx, dres)
//
// ReLU mask: bn_apply_kernel also stores one bit per element (mask[M][C/8], bit = bf16 y > 0), so the backward reads one
// byte per row and thread instead of the 16-byte y vector.  Downsampling blocks run their two BatchNorms
// relu(bn2(c2) + bn_sc(s)) as one pass each way (bn_apply_kernel<true>, bn_bwd_reduce_kernel<3, true>,
// bn_bwd_apply_dual_kernel): no y_sc or dres round trip through memory, and both layers' results equal the two-layer path's.
//
// Reference counterpart: nn.BatchNorm2d / F.relu inside src/model_ops/resnet.py:14-64 and vgg.py:46-59 (PyTorch-0.3 CPU).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr int BN_THREADS = 512;
constexpr int BN_VEC = 8;                      // channels per thread (one 16-byte access)
constexpr int BN_UNROLL = 4;

struct BnFwdArgs {
  const __nv_bfloat16* x;         // [M][C]
  const __nv_bfloat16* res;       // optional residual [M][C]
  __nv_bfloat16* y;               // [M][C]
  const float* gamma;             // [C]
  const float* beta;              // [C]
  float* running_mean;            // [C] (may be null)
  float* running_var;
  float* mean;                    // [C] saved for backward (written by the statistics kernel, read by apply)
  float* invstd;                  // [C]
  float* partial;                 // [grid][2][C] workspace (statistics kernel)
  unsigned int* counter;          // zero on entry, reset by the last CTA
  long long M;
  int C;
  int rows_per_cta;
  float eps, momentum;
  int relu;
};

// bn_apply_kernel only (a parameter of its own: BnFwdArgs, which bn_stats_kernel takes too, stays as it was)
struct BnApplyArgs {
  uint8_t* mask;                  // optional [M][C/8]: bit i of byte (row, cv) = (bf16 y > 0) for channel 8*cv + i
  // downsampling-block pair (bn_apply_kernel<true>): the residual is a second BatchNorm's output bf16(res * scale_s + shift_s),
  // formed here from the raw shortcut convolution output in `res` instead of being read back from memory
  const float* gamma_s;
  const float* beta_s;
  const float* mean_s;
  const float* invstd_s;
};

struct BnBwdArgs {
  const __nv_bfloat16* dy;        // [M][C]
  const __nv_bfloat16* y;         // forward output (ReLU mask); null when relu == 0 -- or when the mask is recomputed from x
  const float* beta;              // relu && !y: mask = (bf16(fma(x, gamma*invstd, beta - mean*gamma*invstd)) > 0), the forward's own
                                  // arithmetic (layers without a residual input) -- one tensor less to read in both kernels
  const __nv_bfloat16* x;         // [M][C]
  const float* gamma;
  const float* mean;
  const float* invstd;
  __nv_bfloat16* dx;              // [M][C]
  __nv_bfloat16* dres;            // optional: gradient of the residual input
  float* dgamma;                  // [C]
  float* dbeta;                   // [C]
  float* partial;                 // [grid][2][C]
  float* sums;                    // [2][C] : mean(dy_r), mean(dy_r * xhat)
  unsigned int* counter;
  long long M;
  int C;
  int rows_per_cta;
  int relu;
  const uint8_t* mask;            // MASK == 3: the forward's ReLU bits [M][C/8]
  // downsampling-block pair (dual kernels): the shortcut BatchNorm, whose input xs sees the same masked gradient dz
  const __nv_bfloat16* xs;        // [M][C]
  const float* gamma_s;
  const float* mean_s;
  const float* invstd_s;
  __nv_bfloat16* dxs;             // [M][C]
  float* dgamma_s;
  float* dbeta_s;
  float* sums_s;                  // [2][C]
};

__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
  const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 a = __bfloat1622float2(p[i]); f[2 * i] = a.x; f[2 * i + 1] = a.y; }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 v;
  __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) p[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return v;
}
// did the forward's BatchNorm + ReLU output survive?  Same fp32 arithmetic and the same bf16 rounding as bn_apply_kernel.
__device__ __forceinline__ bool relu_mask(float x, float scale, float shift) {
  return __bfloat162float(__float2bfloat16_rn(fmaf(x, scale, shift))) > 0.f;
}
__device__ __forceinline__ uint4 ldg16(const __nv_bfloat16* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

// ReLU bits of one row's 8 channels as stored: bit i = (bf16 value i of v) > 0
__device__ __forceinline__ uint32_t pos_bits8(const uint4& v) {
  float f[BN_VEC];
  unpack8(v, f);
  uint32_t b = 0;
#pragma unroll
  for (int i = 0; i < BN_VEC; ++i) b |= (f[i] > 0.f ? 1u : 0u) << i;
  return b;
}
__device__ __forceinline__ uint32_t ldg_u8(const uint8_t* p) {
  uint16_t v;
  asm volatile("ld.global.nc.L1::no_allocate.u8 %0, [%1];" : "=h"(v) : "l"(p));
  return v;
}
// the shortcut BatchNorm's output value as the unpaired layer stores it: bf16(fma(x, scale, shift))
__device__ __forceinline__ float bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

extern __shared__ __align__(16) float bn_smem[];

// CTA-level fold of the per-thread accumulators acc[2][8] over the row groups, then this CTA's partial[2][C] (fixed order).
// NA accumulator rows (2, or 3 for the downsampling pair); every index is folded in the same order whatever NA is.
template <int NA>
__device__ __forceinline__ void cta_fold(const float (&acc)[NA][BN_VEC], float* partial_blk, int C, int rgroups, int rg, int cv) {
  // smem layout: [rgroups][NA][C]  (rgroups * NA * C == BN_THREADS * 8 * NA floats = 16 KB * NA)
#pragma unroll
  for (int a = 0; a < NA; ++a) {
    float4* dst = reinterpret_cast<float4*>(&bn_smem[(rg * NA + a) * C + cv * BN_VEC]);
    dst[0] = make_float4(acc[a][0], acc[a][1], acc[a][2], acc[a][3]);
    dst[1] = make_float4(acc[a][4], acc[a][5], acc[a][6], acc[a][7]);
  }
  __syncthreads();
  const int n_idx = NA * C;
  for (int idx = threadIdx.x; idx < n_idx; idx += BN_THREADS) {
    float s0 = 0.f, s1 = 0.f;
    int g = 0;
    for (; g + 1 < rgroups; g += 2) { s0 += bn_smem[g * n_idx + idx]; s1 += bn_smem[(g + 1) * n_idx + idx]; }
    if (g < rgroups) s0 += bn_smem[g * n_idx + idx];
    partial_blk[idx] = s0 + s1;
  }
}

__device__ __forceinline__ bool last_cta(unsigned int* counter) {
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    // release the CTA's partial (ordered before this thread by the barrier) with the ticket, acquire everybody else's
    unsigned int prev;
    asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(prev) : "l"(counter) : "memory");
    s_last = (prev == gridDim.x - 1);
    if (s_last) *counter = 0;
  }
  __syncthreads();
  return s_last != 0;
}

// Grid-level fold by the last CTA: totals[idx] = sum_b partial[b][first + idx], idx in [0, 2C), each CTA's partial NA * C floats:
// 16-byte loads, the CTAs' partials split into interleaved subsets that are combined in a fixed order (which depends on C and
// the grid only, so a 2C window of a 3-row partial folds exactly as a 2-row partial would).  Result in bn_smem[0 .. 2C).
template <int NA>
__device__ __forceinline__ void grid_fold(const float* partial, int C, int first = 0) {
  const int items4 = (2 * C) >> 2;
  const int stride4 = (NA * C) >> 2;
  const int nblk = (int)gridDim.x;
  const float4* p4 = reinterpret_cast<const float4*>(partial + first);
  float4* s4 = reinterpret_cast<float4*>(bn_smem);
  __syncthreads();
  if (items4 <= BN_THREADS) {
    const int SUB = BN_THREADS / items4;
    const int item = threadIdx.x % items4, sub = threadIdx.x / items4;
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    if (sub < SUB) {
      constexpr int FB = 16;                                        // independent 16-byte loads in flight
      for (int g0 = sub; g0 < nblk; g0 += FB * SUB) {
        float4 v[FB];
#pragma unroll
        for (int u = 0; u < FB; ++u) {
          const int g = g0 + u * SUB;
          v[u] = g < nblk ? __ldcg(p4 + (long long)g * stride4 + item) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < FB; ++u) { t.x += v[u].x; t.y += v[u].y; t.z += v[u].z; t.w += v[u].w; }    // fixed order
      }
    }
    s4[items4 + threadIdx.x] = t;                                  // scratch behind the totals
    __syncthreads();
    if (sub == 0) {
      float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int s2 = 0; s2 < SUB; ++s2) {
        const float4 v = s4[items4 + s2 * items4 + item];
        tot.x += v.x; tot.y += v.y; tot.z += v.z; tot.w += v.w;
      }
      s4[item] = tot;
    }
  } else {
    for (int item = threadIdx.x; item < items4; item += BN_THREADS) {
      float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0;
      int g = 0;
      for (; g + 1 < nblk; g += 2) {
        const float4 v0 = __ldcg(p4 + (long long)g * stride4 + item), v1 = __ldcg(p4 + (long long)(g + 1) * stride4 + item);
        a0.x += v0.x; a0.y += v0.y; a0.z += v0.z; a0.w += v0.w;
        a1.x += v1.x; a1.y += v1.y; a1.z += v1.z; a1.w += v1.w;
      }
      if (g < nblk) { const float4 v0 = __ldcg(p4 + (long long)g * stride4 + item); a0.x += v0.x; a0.y += v0.y; a0.z += v0.z; a0.w += v0.w; }
      s4[item] = make_float4(a0.x + a1.x, a0.y + a1.y, a0.z + a1.z, a0.w + a1.w);
    }
  }
  __syncthreads();
}

// rows [r0, r1) of this CTA, row groups interleaved, UNROLL independent rows in flight per thread
#define BN_ROW_LOOP(BODY_LOAD, BODY_USE) BN_ROW_LOOP_U(BN_UNROLL, BODY_LOAD, BODY_USE)
#define BN_ROW_LOOP_U(UNROLL, BODY_LOAD, BODY_USE)                                                  \
  {                                                                                                 \
    long long r = r0 + rg;                                                                          \
    for (; r + (long long)(UNROLL - 1) * rgroups < r1; r += (long long)UNROLL * rgroups) {          \
      _Pragma("unroll") for (int u = 0; u < UNROLL; ++u) { const long long off = (r + (long long)u * rgroups) * a.C + cv * BN_VEC; BODY_LOAD }  \
      _Pragma("unroll") for (int u = 0; u < UNROLL; ++u) { const long long off = (r + (long long)u * rgroups) * a.C + cv * BN_VEC; BODY_USE }   \
    }                                                                                               \
    for (; r < r1; r += rgroups) {                                                                  \
      const int u = 0; const long long off = r * a.C + cv * BN_VEC; BODY_LOAD BODY_USE              \
    }                                                                                               \
  }

__global__ void __launch_bounds__(BN_THREADS, 2) bn_stats_kernel(const BnFwdArgs a) {
  const int tpc = a.C / BN_VEC;
  const int rgroups = BN_THREADS / tpc;
  const int cv = threadIdx.x % tpc, rg = threadIdx.x / tpc;
  const long long r0 = (long long)blockIdx.x * a.rows_per_cta;
  long long r1 = r0 + a.rows_per_cta; if (r1 > a.M) r1 = a.M;
  float acc[2][BN_VEC];
#pragma unroll
  for (int i = 0; i < BN_VEC; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
  uint4 xv[BN_UNROLL];
  BN_ROW_LOOP(
      { xv[u] = ldg16(a.x + off); },
      { float f[BN_VEC]; unpack8(xv[u], f);
        _Pragma("unroll") for (int i = 0; i < BN_VEC; ++i) { acc[0][i] += f[i]; acc[1][i] = fmaf(f[i], f[i], acc[1][i]); } (void)off; })
  cta_fold<2>(acc, a.partial + (long long)blockIdx.x * 2 * a.C, a.C, rgroups, rg, cv);
  if (last_cta(a.counter)) {
    grid_fold<2>(a.partial, a.C);
    const float inv_m = 1.0f / (float)a.M;
    for (int c = threadIdx.x; c < a.C; c += BN_THREADS) {
      const float m = bn_smem[c] * inv_m;
      float var = fmaf(-m, m, bn_smem[a.C + c] * inv_m);
      var = var < 0.f ? 0.f : var;
      a.mean[c] = m;
      a.invstd[c] = rsqrtf(var + a.eps);
      if (a.running_mean) {
        // __fmul_rn: rounded on its own, never contracted into the fma below (the conv epilogue's finalisation does the same,
        // so both paths update the running variance bit-identically)
        const float unbiased = a.M > 1 ? __fmul_rn(var, (float)a.M / (float)(a.M - 1)) : var;
        a.running_mean[c] = fmaf(a.momentum, m - a.running_mean[c], a.running_mean[c]);
        a.running_var[c] = fmaf(a.momentum, unbiased - a.running_var[c], a.running_var[c]);
      }
    }
  }
}

// Scale / shift per channel sit in shared memory (fwd_smem_bytes: [2][C] floats, [4][C] with DUAL), so the shortcut layer's
// coefficients add no registers.
// DUAL: y = relu?(bn(x) + bf16(bn_s(res))) for a downsampling block, the shortcut BatchNorm's output formed from its raw input.
template <bool DUAL>
__global__ void __launch_bounds__(BN_THREADS, 2) bn_apply_kernel(const BnFwdArgs a, const BnApplyArgs p) {
  const int tpc = a.C / BN_VEC;
  const int rgroups = BN_THREADS / tpc;
  const int cv = threadIdx.x % tpc, rg = threadIdx.x / tpc;
  for (int c = threadIdx.x; c < a.C; c += BN_THREADS) {
    const float sc = a.gamma[c] * a.invstd[c];
    bn_smem[c] = sc;
    bn_smem[a.C + c] = fmaf(-a.mean[c], sc, a.beta[c]);
    if (DUAL) {
      const float scs = p.gamma_s[c] * p.invstd_s[c];
      bn_smem[2 * a.C + c] = scs;
      bn_smem[3 * a.C + c] = fmaf(-p.mean_s[c], scs, p.beta_s[c]);
    }
  }
  __syncthreads();
  const float* scale = bn_smem + cv * BN_VEC;
  const float* shift = scale + a.C;
  const float* sc_s = shift + a.C;
  const float* sh_s = sc_s + a.C;
  const long long r0 = (long long)blockIdx.x * a.rows_per_cta;
  long long r1 = r0 + a.rows_per_cta; if (r1 > a.M) r1 = a.M;
  constexpr int AU = DUAL ? 1 : 2;                                 // rows in flight per thread that fit 64 registers
  uint4 xv[AU], rv[AU];
  const bool has_res = a.res != nullptr;
  BN_ROW_LOOP_U(AU,
      { xv[u] = ldg16(a.x + off); if (has_res) rv[u] = ldg16(a.res + off); },
      { float f[BN_VEC]; unpack8(xv[u], f);
        _Pragma("unroll") for (int i = 0; i < BN_VEC; ++i) f[i] = fmaf(f[i], scale[i], shift[i]);
        if (has_res) { float g[BN_VEC]; unpack8(rv[u], g);
          if (DUAL) { _Pragma("unroll") for (int i = 0; i < BN_VEC; ++i) g[i] = bf16_round(fmaf(g[i], sc_s[i], sh_s[i])); }
          _Pragma("unroll") for (int i = 0; i < BN_VEC; ++i) f[i] += g[i]; }
        if (a.relu) { _Pragma("unroll") for (int i = 0; i < BN_VEC; ++i) f[i] = fmaxf(f[i], 0.f); }
        const uint4 yv = pack8(f);
        *reinterpret_cast<uint4*>(a.y + off) = yv;
        if (p.mask) p.mask[off >> 3] = (uint8_t)pos_bits8(yv); })                  // off / 8 == row * C / 8 + cv
}

// MASK: 0 = no ReLU, 1 = ReLU mask from the saved output y, 2 = mask recomputed from x (specialised: the apply kernel has to fit
// 64 registers for two CTAs per SM), 3 = the forward's ReLU bits (one byte per row and thread instead of 16).
// DUAL (MASK == 3): the downsampling pair -- a third accumulator row sum(dz * xhat_s) over the shortcut input xs, with the
// same rows, order and grid as the unpaired layers, so both layers' dgamma / dbeta equal their separate reductions bit for bit.
template <int MASK, bool DUAL = false>
__global__ void __launch_bounds__(BN_THREADS) bn_bwd_reduce_kernel(const BnBwdArgs a) {
  constexpr int NA = DUAL ? 3 : 2;
  const int tpc = a.C / BN_VEC;
  const int rgroups = BN_THREADS / tpc;
  const int cv = threadIdx.x % tpc, rg = threadIdx.x / tpc;
  float mean[BN_VEC], istd[BN_VEC], mean_s[BN_VEC], istd_s[BN_VEC];
#pragma unroll
  for (int i = 0; i < BN_VEC; ++i) { mean[i] = a.mean[cv * BN_VEC + i]; istd[i] = a.invstd[cv * BN_VEC + i]; }
  if (DUAL) {
#pragma unroll
    for (int i = 0; i < BN_VEC; ++i) { mean_s[i] = a.mean_s[cv * BN_VEC + i]; istd_s[i] = a.invstd_s[cv * BN_VEC + i]; }
  }
  const long long r0 = (long long)blockIdx.x * a.rows_per_cta;
  long long r1 = r0 + a.rows_per_cta; if (r1 > a.M) r1 = a.M;
  float acc[NA][BN_VEC];
#pragma unroll
  for (int i = 0; i < BN_VEC; ++i) {
#pragma unroll
    for (int k = 0; k < NA; ++k) acc[k][i] = 0.f;
  }
  uint4 dv[BN_UNROLL], xv[BN_UNROLL], yv[BN_UNROLL], sv[BN_UNROLL];
  uint32_t mv[BN_UNROLL];
  constexpr bool relu_y = MASK == 1, relu_x = MASK == 2, relu_b = MASK == 3;
  float sc[BN_VEC], sh[BN_VEC];
#pragma unroll
  for (int i = 0; i < BN_VEC; ++i) {
    sc[i] = relu_x ? a.gamma[cv * BN_VEC + i] * istd[i] : 0.f;
    sh[i] = relu_x ? fmaf(-mean[i], sc[i], a.beta[cv * BN_VEC + i]) : 0.f;
  }
  BN_ROW_LOOP(
      { dv[u] = ldg16(a.dy + off); xv[u] = ldg16(a.x + off); if (relu_y) yv[u] = ldg16(a.y + off);
        if (relu_b) mv[u] = ldg_u8(a.mask + (off >> 3)); if (DUAL) sv[u] = ldg16(a.xs + off); },
      { float d[BN_VEC]; float xf[BN_VEC]; unpack8(dv[u], d); unpack8(xv[u], xf);
        if (relu_y) { float yf[BN_VEC]; unpack8(yv[u], yf); _Pragma("unroll") for (int i = 0; i < BN_VEC; ++i) d[i] = yf[i] > 0.f ? d[i] : 0.f; }
        if (relu_x) { _Pragma("unroll") for (int i = 0; i < BN_VEC; ++i) d[i] = relu_mask(xf[i], sc[i], sh[i]) ? d[i] : 0.f; }
        if (relu_b) { _Pragma("unroll") for (int i = 0; i < BN_VEC; ++i) d[i] = (mv[u] >> i) & 1u ? d[i] : 0.f; }
        _Pragma("unroll") for (int i = 0; i < BN_VEC; ++i) { acc[0][i] += d[i]; acc[1][i] = fmaf(d[i], (xf[i] - mean[i]) * istd[i], acc[1][i]); }
        if (DUAL) { float sf[BN_VEC]; unpack8(sv[u], sf);
          _Pragma("unroll") for (int i = 0; i < BN_VEC; ++i) acc[NA - 1][i] = fmaf(d[i], (sf[i] - mean_s[i]) * istd_s[i], acc[NA - 1][i]); }
        (void)off; })
  cta_fold<NA>(acc, a.partial + (long long)blockIdx.x * NA * a.C, a.C, rgroups, rg, cv);
  if (last_cta(a.counter)) {
    grid_fold<NA>(a.partial, a.C);
    const float inv_m = 1.0f / (float)a.M;
    for (int c = threadIdx.x; c < a.C; c += BN_THREADS) {
      const float s = bn_smem[c], q = bn_smem[a.C + c];
      a.dbeta[c] = s;
      a.dgamma[c] = q;
      a.sums[c] = s * inv_m;
      a.sums[a.C + c] = q * inv_m;
      if (DUAL) { a.dbeta_s[c] = s; a.sums_s[c] = s * inv_m; }          // both layers see the same dz
    }
    if (DUAL) {
      grid_fold<NA>(a.partial, a.C, a.C);                              // rows 1, 2: sum(dz * xhat_s) lands in bn_smem[C .. 2C)
      for (int c = threadIdx.x; c < a.C; c += BN_THREADS) {
        const float q = bn_smem[a.C + c];
        a.dgamma_s[c] = q;
        a.sums_s[a.C + c] = q * inv_m;
      }
    }
  }
}

template <int MASK>
__global__ void __launch_bounds__(BN_THREADS, 2) bn_bwd_apply_kernel(const BnBwdArgs a) {
  const int tpc = a.C / BN_VEC;
  const int rgroups = BN_THREADS / tpc;
  const int cv = threadIdx.x % tpc, rg = threadIdx.x / tpc;
  // dx = gs * (d - m1 - xhat * m2) with xhat = (x - mean) * istd   ==   A * d + B * x + Cc
  float cA[BN_VEC], cB[BN_VEC], cC[BN_VEC];
  constexpr bool relu_y = MASK == 1, relu_x = MASK == 2, relu_b = MASK == 3;
  __shared__ __align__(16) float s_sh[BN_THREADS * BN_VEC];           // the forward's shift per channel (mask recomputation), read per row: keeps
  if (relu_x) {                                        // the kernel inside 64 registers
    for (int c = threadIdx.x; c < a.C; c += BN_THREADS) s_sh[c] = fmaf(-a.mean[c], a.gamma[c] * a.invstd[c], a.beta[c]);
    __syncthreads();
  }
  const float* sh = s_sh + cv * BN_VEC;
#pragma unroll
  for (int i = 0; i < BN_VEC; ++i) {
    const int c = cv * BN_VEC + i;
    const float istd = a.invstd[c], gs = a.gamma[c] * istd, m1 = a.sums[c], m2 = a.sums[a.C + c], mean = a.mean[c];
    cA[i] = gs;                                        // == the forward's scale
    // every rounding stated (tests/exact_ref.py restates them): cB is two products and nothing to contract; cC's inner term is
    // one fma of the rounded m2 * istd, which is the contraction nvcc chose for the unfused spelling
    cB[i] = -gs * m2 * istd;
    cC[i] = __fmul_rn(gs, fmaf(__fmul_rn(m2, istd), mean, -m1));
  }
  const long long r0 = (long long)blockIdx.x * a.rows_per_cta;
  long long r1 = r0 + a.rows_per_cta; if (r1 > a.M) r1 = a.M;
  // three streams in flight: keep the register count moderate (the bit mask's row offset arithmetic tips two rows over 64)
  constexpr int BU = relu_b ? 1 : 2;
  long long r = r0 + rg;
  for (; r + (long long)(BU - 1) * rgroups < r1; r += (long long)BU * rgroups) {
    uint4 dv[BU], xv[BU], yv[BU];
    uint32_t mv[BU];
#pragma unroll
    for (int u = 0; u < BU; ++u) {
      const long long off = (r + (long long)u * rgroups) * a.C + cv * BN_VEC;
      dv[u] = ldg16(a.dy + off); xv[u] = ldg16(a.x + off); if (relu_y) yv[u] = ldg16(a.y + off);
      if (relu_b) mv[u] = ldg_u8(a.mask + (off >> 3));
    }
#pragma unroll
    for (int u = 0; u < BU; ++u) {
      const long long off = (r + (long long)u * rgroups) * a.C + cv * BN_VEC;
      float d[BN_VEC], xf[BN_VEC];
      unpack8(dv[u], d); unpack8(xv[u], xf);
      if (relu_y) { float yf[BN_VEC]; unpack8(yv[u], yf);
#pragma unroll
        for (int i = 0; i < BN_VEC; ++i) d[i] = yf[i] > 0.f ? d[i] : 0.f; }
      if (relu_x) {
#pragma unroll
        for (int i = 0; i < BN_VEC; ++i) d[i] = relu_mask(xf[i], cA[i], sh[i]) ? d[i] : 0.f; }
      if (relu_b) {
#pragma unroll
        for (int i = 0; i < BN_VEC; ++i) d[i] = (mv[u] >> i) & 1u ? d[i] : 0.f; }
      if (a.dres) *reinterpret_cast<uint4*>(a.dres + off) = pack8(d);
      float o[BN_VEC];
#pragma unroll
      for (int i = 0; i < BN_VEC; ++i) o[i] = fmaf(cA[i], d[i], fmaf(cB[i], xf[i], cC[i]));
      *reinterpret_cast<uint4*>(a.dx + off) = pack8(o);
    }
  }
  for (; r < r1; r += rgroups) {
    const long long off = r * a.C + cv * BN_VEC;
    float d[BN_VEC], xf[BN_VEC];
    const uint4 dvv = ldg16(a.dy + off), xvv = ldg16(a.x + off);
    unpack8(dvv, d); unpack8(xvv, xf);
    if (relu_y) { float yf[BN_VEC]; const uint4 yvv = ldg16(a.y + off); unpack8(yvv, yf);
#pragma unroll
      for (int i = 0; i < BN_VEC; ++i) d[i] = yf[i] > 0.f ? d[i] : 0.f; }
    if (relu_x) {
#pragma unroll
      for (int i = 0; i < BN_VEC; ++i) d[i] = relu_mask(xf[i], cA[i], sh[i]) ? d[i] : 0.f; }
    if (relu_b) { const uint32_t m = ldg_u8(a.mask + (off >> 3));
#pragma unroll
      for (int i = 0; i < BN_VEC; ++i) d[i] = (m >> i) & 1u ? d[i] : 0.f; }
    if (a.dres) *reinterpret_cast<uint4*>(a.dres + off) = pack8(d);
    float o[BN_VEC];
#pragma unroll
    for (int i = 0; i < BN_VEC; ++i) o[i] = fmaf(cA[i], d[i], fmaf(cB[i], xf[i], cC[i]));
    *reinterpret_cast<uint4*>(a.dx + off) = pack8(o);
  }
}

// Downsampling pair: dz = mask(dy) -> dx = A * dz + B * x + Cc (bn2) and dxs = As * dz + Bs * xs + Cs (shortcut BatchNorm), the
// coefficients formed exactly as bn_bwd_apply_kernel forms them.  The shortcut's sit in shared memory (3C floats of dynamic
// smem, read per row) and one row is in flight per thread: three input streams and two outputs inside 64 registers.
__global__ void __launch_bounds__(BN_THREADS, 2) bn_bwd_apply_dual_kernel(const BnBwdArgs a) {
  const int tpc = a.C / BN_VEC;
  const int rgroups = BN_THREADS / tpc;
  const int cv = threadIdx.x % tpc, rg = threadIdx.x / tpc;
  for (int c = threadIdx.x; c < a.C; c += BN_THREADS) {
    const float istd = a.invstd_s[c], gs = a.gamma_s[c] * istd, m1 = a.sums_s[c], m2 = a.sums_s[a.C + c], mean = a.mean_s[c];
    bn_smem[c] = gs;
    bn_smem[a.C + c] = -gs * m2 * istd;
    bn_smem[2 * a.C + c] = __fmul_rn(gs, fmaf(__fmul_rn(m2, istd), mean, -m1));
  }
  float cA[BN_VEC], cB[BN_VEC], cC[BN_VEC];
#pragma unroll
  for (int i = 0; i < BN_VEC; ++i) {
    const int c = cv * BN_VEC + i;
    const float istd = a.invstd[c], gs = a.gamma[c] * istd, m1 = a.sums[c], m2 = a.sums[a.C + c], mean = a.mean[c];
    cA[i] = gs;
    cB[i] = -gs * m2 * istd;
    cC[i] = __fmul_rn(gs, fmaf(__fmul_rn(m2, istd), mean, -m1));
  }
  __syncthreads();
  const float* sA = bn_smem + cv * BN_VEC;
  const float* sB = sA + a.C;
  const float* sC = sB + a.C;
  const long long r0 = (long long)blockIdx.x * a.rows_per_cta;
  long long r1 = r0 + a.rows_per_cta; if (r1 > a.M) r1 = a.M;
  for (long long r = r0 + rg; r < r1; r += rgroups) {
    const long long off = r * a.C + cv * BN_VEC;
    const uint4 dvv = ldg16(a.dy + off), xvv = ldg16(a.x + off), svv = ldg16(a.xs + off);
    const uint32_t m = ldg_u8(a.mask + (off >> 3));
    float d[BN_VEC], f[BN_VEC], o[BN_VEC];
    unpack8(dvv, d);
#pragma unroll
    for (int i = 0; i < BN_VEC; ++i) d[i] = (m >> i) & 1u ? d[i] : 0.f;
    unpack8(xvv, f);
#pragma unroll
    for (int i = 0; i < BN_VEC; ++i) o[i] = fmaf(cA[i], d[i], fmaf(cB[i], f[i], cC[i]));
    *reinterpret_cast<uint4*>(a.dx + off) = pack8(o);
    unpack8(svv, f);
#pragma unroll
    for (int i = 0; i < BN_VEC; ++i) o[i] = fmaf(sA[i], d[i], fmaf(sB[i], f[i], sC[i]));
    *reinterpret_cast<uint4*>(a.dxs + off) = pack8(o);
  }
}

// C / 8 vector lanes must tile the 512-thread CTA
bool supported(int C) { return C >= BN_VEC && C % BN_VEC == 0 && BN_THREADS % (C / BN_VEC) == 0; }

// Grid / rows per CTA.  `reduce`: every CTA adds a partial the last CTA has to fold, so the grid is capped at the SM count;
// streaming kernels go up to 4 CTAs per SM (one CTA per ~32 KB of the tensor).
int plan_rows(long long M, int C, int num_sms, bool reduce, int* grid) {
  const int rgroups = BN_THREADS / (C / BN_VEC);
  const long long bytes = M * (long long)C * 2;
  long long target = (bytes + 32767) / 32768;
  const long long cap = reduce ? num_sms : 4LL * num_sms;
  if (target > cap) target = cap;
  if (target < 1) target = 1;
  long long rows = (M + target - 1) / target;
  rows = (rows + rgroups - 1) / rgroups * rgroups;
  if (rows < rgroups) rows = rgroups;
  *grid = (int)((M + rows - 1) / rows);
  return (int)rows;
}

size_t smem_bytes(int C, int na = 2) {
  // cta_fold: BN_THREADS * 8 * na floats (32 KB, 48 KB for the pair); grid_fold: totals 2C floats + BN_THREADS float4 of scratch
  size_t a = (size_t)BN_THREADS * na * BN_VEC * sizeof(float);
  size_t b = ((size_t)2 * C + 4 * BN_THREADS) * sizeof(float);
  return a > b ? a : b;
}

// bn_apply_kernel's per-channel coefficients; C = 4096 with DUAL needs 64 KB (opted in once per process)
size_t fwd_smem_bytes(int C, bool dual) {
  const size_t b = (size_t)(dual ? 4 : 2) * C * sizeof(float);
  if (dual && b > 48 * 1024) {
    static const bool once = [] {
      cudaFuncSetAttribute(bn_apply_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 4096 * (int)sizeof(float));
      return true;
    }();
    (void)once;
  }
  return b;
}

}  // namespace

extern "C" int drc_bn_supported(int C) { return supported(C) ? 1 : 0; }

// workspace floats needed for `partial` (the downsampling pair's backward needs 3/2 of it)
extern "C" long long drc_bn_workspace(long long M, int C, int num_sms) {
  if (!supported(C)) return -1;
  int grid; plan_rows(M, C, num_sms, true, &grid);
  return (long long)grid * 2 * C;
}

// Forward.  have_stats != 0: mean / invstd were produced by the convolution epilogue -> only the apply kernel runs.
// mask (optional, relu only): the ReLU bits [M][C/8] for the backward's MASK == 3.
extern "C" int drc_bn_fwd(const void* x, const void* res, void* y, void* mask, const float* gamma, const float* beta, float* running_mean,
                          float* running_var, float* mean, float* invstd, float* partial, unsigned int* counter, long long M, int C,
                          float eps, float momentum, int relu, int num_sms, int have_stats, cudaStream_t stream) {
  if (!supported(C)) return -1;
  BnFwdArgs a;
  a.x = (const __nv_bfloat16*)x; a.res = (const __nv_bfloat16*)res; a.y = (__nv_bfloat16*)y; a.gamma = gamma; a.beta = beta;
  a.running_mean = running_mean; a.running_var = running_var; a.mean = mean; a.invstd = invstd; a.partial = partial;
  a.counter = counter; a.M = M; a.C = C; a.eps = eps; a.momentum = momentum; a.relu = relu;
  BnApplyArgs p = {};
  p.mask = relu ? (uint8_t*)mask : nullptr;
  int grid;
  if (!have_stats) {
    a.rows_per_cta = plan_rows(M, C, num_sms, true, &grid);
    bn_stats_kernel<<<grid, BN_THREADS, smem_bytes(C), stream>>>(a);
  }
  a.rows_per_cta = plan_rows(M, C, num_sms, false, &grid);
  bn_apply_kernel<false><<<grid, BN_THREADS, fwd_smem_bytes(C, false), stream>>>(a, p);
  return (int)cudaGetLastError();
}

// Forward of a downsampling block's pair: y = relu(bn(x) + bn_s(xs)) in one pass, both layers' statistics from their
// convolutions' epilogues.  Same values as drc_bn_fwd(xs) followed by drc_bn_fwd(x, residual = that output).
extern "C" int drc_bn_fwd_dual(const void* x, const void* xs, void* y, void* mask, const float* gamma, const float* beta,
                               const float* mean, const float* invstd, const float* gamma_s, const float* beta_s,
                               const float* mean_s, const float* invstd_s, long long M, int C, int num_sms, cudaStream_t stream) {
  if (!supported(C) || !mask) return -1;
  BnFwdArgs a;
  a.x = (const __nv_bfloat16*)x; a.res = (const __nv_bfloat16*)xs; a.y = (__nv_bfloat16*)y; a.gamma = gamma; a.beta = beta;
  a.running_mean = a.running_var = nullptr; a.mean = const_cast<float*>(mean); a.invstd = const_cast<float*>(invstd);
  a.partial = nullptr; a.counter = nullptr; a.M = M; a.C = C; a.eps = 0.f; a.momentum = 0.f; a.relu = 1;
  BnApplyArgs p;
  p.mask = (uint8_t*)mask; p.gamma_s = gamma_s; p.beta_s = beta_s; p.mean_s = mean_s; p.invstd_s = invstd_s;
  int grid;
  a.rows_per_cta = plan_rows(M, C, num_sms, false, &grid);
  bn_apply_kernel<true><<<grid, BN_THREADS, fwd_smem_bytes(C, true), stream>>>(a, p);
  return (int)cudaGetLastError();
}

// mask_mode: 0 = no ReLU, 1 = mask from the saved output y, 2 = recomputed from x (needs beta), 3 = the forward's bits `mask`
extern "C" int drc_bn_bwd(const void* dy, const void* y, const void* mask, const void* x, const float* gamma, const float* beta,
                          const float* mean, const float* invstd,
                          void* dx, void* dres, float* dgamma, float* dbeta, float* partial, float* sums, unsigned int* counter,
                          long long M, int C, int mask_mode, int num_sms, cudaStream_t stream) {
  if (!supported(C)) return -1;
  if ((mask_mode == 1 && !y) || (mask_mode == 2 && !beta) || (mask_mode == 3 && !mask) || mask_mode < 0 || mask_mode > 3) return -2;
  BnBwdArgs a = {};
  a.dy = (const __nv_bfloat16*)dy; a.y = (const __nv_bfloat16*)y; a.x = (const __nv_bfloat16*)x; a.gamma = gamma; a.beta = beta;
  a.mean = mean; a.invstd = invstd; a.mask = (const uint8_t*)mask;
  a.dx = (__nv_bfloat16*)dx; a.dres = (__nv_bfloat16*)dres; a.dgamma = dgamma; a.dbeta = dbeta;
  a.partial = partial; a.sums = sums; a.counter = counter; a.M = M; a.C = C; a.relu = mask_mode != 0;
  int grid;
  a.rows_per_cta = plan_rows(M, C, num_sms, true, &grid);
  if (mask_mode == 0) bn_bwd_reduce_kernel<0><<<grid, BN_THREADS, smem_bytes(C), stream>>>(a);
  else if (mask_mode == 1) bn_bwd_reduce_kernel<1><<<grid, BN_THREADS, smem_bytes(C), stream>>>(a);
  else if (mask_mode == 2) bn_bwd_reduce_kernel<2><<<grid, BN_THREADS, smem_bytes(C), stream>>>(a);
  else bn_bwd_reduce_kernel<3><<<grid, BN_THREADS, smem_bytes(C), stream>>>(a);
  a.rows_per_cta = plan_rows(M, C, num_sms, false, &grid);
  if (mask_mode == 0) bn_bwd_apply_kernel<0><<<grid, BN_THREADS, 0, stream>>>(a);
  else if (mask_mode == 1) bn_bwd_apply_kernel<1><<<grid, BN_THREADS, 0, stream>>>(a);
  else if (mask_mode == 2) bn_bwd_apply_kernel<2><<<grid, BN_THREADS, 0, stream>>>(a);
  else bn_bwd_apply_kernel<3><<<grid, BN_THREADS, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

// Backward of the downsampling pair (the forward's bits `mask`): one reduce for both layers' sums (partial: 3/2 of
// drc_bn_workspace, sums and sums_s [2][C] each), one apply writing dx and dxs.  Bit-identical to drc_bn_bwd(mode 3, dres)
// for the main layer followed by drc_bn_bwd(dres, mode 0) for the shortcut layer.
extern "C" int drc_bn_bwd_dual(const void* dy, const void* mask, const void* x, const void* xs, const float* gamma,
                               const float* mean, const float* invstd, const float* gamma_s, const float* mean_s,
                               const float* invstd_s, void* dx, void* dxs, float* dgamma, float* dbeta, float* dgamma_s,
                               float* dbeta_s, float* partial, float* sums, float* sums_s, unsigned int* counter, long long M,
                               int C, int num_sms, cudaStream_t stream) {
  if (!supported(C) || !mask) return -1;
  BnBwdArgs a = {};
  a.dy = (const __nv_bfloat16*)dy; a.mask = (const uint8_t*)mask; a.x = (const __nv_bfloat16*)x; a.xs = (const __nv_bfloat16*)xs;
  a.gamma = gamma; a.mean = mean; a.invstd = invstd; a.gamma_s = gamma_s; a.mean_s = mean_s; a.invstd_s = invstd_s;
  a.dx = (__nv_bfloat16*)dx; a.dxs = (__nv_bfloat16*)dxs; a.dgamma = dgamma; a.dbeta = dbeta; a.dgamma_s = dgamma_s;
  a.dbeta_s = dbeta_s; a.partial = partial; a.sums = sums; a.sums_s = sums_s; a.counter = counter; a.M = M; a.C = C; a.relu = 1;
  int grid;
  a.rows_per_cta = plan_rows(M, C, num_sms, true, &grid);
  // 48 KB of dynamic shared memory next to the static ticket flag: over the default limit, opted in once per process
  static const int smem_ok = (int)cudaFuncSetAttribute(bn_bwd_reduce_kernel<3, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                       (int)smem_bytes(4096, 3));
  if (smem_ok != 0) return smem_ok;
  bn_bwd_reduce_kernel<3, true><<<grid, BN_THREADS, smem_bytes(C, 3), stream>>>(a);
  a.rows_per_cta = plan_rows(M, C, num_sms, false, &grid);
  bn_bwd_apply_dual_kernel<<<grid, BN_THREADS, 3 * C * sizeof(float), stream>>>(a);
  return (int)cudaGetLastError();
}

// Backward when the reduction already happened in the dgrad epilogue of the convolution that consumed this layer's output
// (conv_epilogue.cuh, BatchNorm-backward mode): dz arrives masked, sums = [mean(dz), mean(dz * xhat)] -> only the apply kernel.
extern "C" int drc_bn_bwd_apply(const void* dz, const void* x, const float* gamma, const float* mean, const float* invstd,
                                const float* sums, void* dx, long long M, int C, int num_sms, cudaStream_t stream) {
  if (!supported(C)) return -1;
  BnBwdArgs a = {};
  a.dy = (const __nv_bfloat16*)dz; a.y = nullptr; a.x = (const __nv_bfloat16*)x; a.gamma = gamma; a.beta = nullptr;
  a.mean = mean; a.invstd = invstd; a.dx = (__nv_bfloat16*)dx; a.dres = nullptr; a.dgamma = nullptr; a.dbeta = nullptr;
  a.partial = nullptr; a.sums = const_cast<float*>(sums); a.counter = nullptr; a.M = M; a.C = C; a.relu = 0;
  int grid;
  a.rows_per_cta = plan_rows(M, C, num_sms, false, &grid);
  bn_bwd_apply_kernel<0><<<grid, BN_THREADS, 0, stream>>>(a);
  return (int)cudaGetLastError();
}
