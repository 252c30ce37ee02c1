// Epilogue shared by the wgmma convolution kernels (conv_tap_wgmma.cu, conv_halo_wgmma.cu).
//
// A finished 128-pixel x BLOCK_N accumulator tile is drained straight from the wgmma fragments of the MMA warpgroup and is
//   1. converted to bf16 (+ bias, + residual, ReLU-backward mask) and written into a shared-memory staging tile in the
//      128B-swizzled layout TMA expects (row = pixel, 16-byte chunk j of row r at chunk j ^ (r & 7)): every thread stores its own
//      column pairs as bf16x2 words, conflict-free, with no hand-over of the accumulators between threads;
//   2. handed to ONE TMA tensor store per 64-channel half (cp.async.bulk.tensor...global.shared::cta, SASS UTMASTG) -- the
//      4-D box mirrors the load box, so partial batches are clipped by the TMA unit and every global write is a full line;
//   3. (optional) reduced per channel for the BatchNorm that follows the convolution: every epilogue thread owns 8 channels
//      (x one row set) of the staged bf16 tile and accumulates sum / sum-of-squares in registers across the tiles of the
//      persistent CTA (flushed into per-warp shared-memory accumulators).  At kernel end each CTA writes its partial [2][C] to a workspace slot and the LAST CTA
//      (atomic ticket) folds the slots in a fixed order with 16-byte loads and finalises mean / invstd / running statistics:
//      the statistics pass of the BatchNorm (one full read of the activation + one launch per layer) disappears.
//
//   4. (dgrad, optional) BatchNorm BACKWARD reduction of the layer that produced this convolution's input: the dgrad output is the
//      gradient of a BatchNorm(+ReLU) output y, so the epilogue masks it with y > 0 (dz), stores dz, and accumulates sum(dz) and
//      sum(dz * xhat) per channel with the same register / partial / ticket machinery -- the reduce kernel of that BatchNorm's
//      backward (one full read of dy, x and y + one launch) disappears and its apply kernel no longer needs the mask.
//
// Determinism: tile -> CTA assignment, in-CTA accumulation order and the slot fold order depend only on the problem shape and
// the grid size, never on timing; replicas of a batch on different GPUs stay bit-identical (the exact-equality vote needs it).
//
// Reference counterpart: nn.Conv2d followed by nn.BatchNorm2d in src/model_ops/resnet.py:19-24, vgg.py:46-59.
#pragma once
#include "wgmma_common.cuh"

namespace convepi {

constexpr int EPI_THREADS = 128;          // warps 4..7 (the MMA warpgroup)
constexpr int EPI_BAR_ID = 1;
constexpr int STAT_MAX_C = 512;

struct BnStatArgs {
  float* partial;                 // [slots][2][C] workspace, null: no statistics
  unsigned int* counter;          // zero on entry, reset by the last CTA
  float* mean;                    // [C] out
  float* invstd;                  // [C] out
  float* running_mean;            // [C] or null
  float* running_var;
  long long count;                // elements per channel (N * OH * OW)
  float eps, momentum;
  // BatchNorm-backward mode (dgrad epilogue): non-null bwd_x switches the reduction to sum(dz), sum(dz * xhat)
  const __nv_bfloat16* bwd_x;     // input x of the BatchNorm whose output fed this convolution (shape of the dgrad output)
  const __nv_bfloat16* bwd_mask;  // that BatchNorm's output y (this convolution's forward input): dz = d * (y > 0); null = no ReLU
  const float* bwd_mean;          // [C] batch statistics of that BatchNorm
  const float* bwd_invstd;
  float* bwd_sums;                // [2][C] out: mean(dz), mean(dz * xhat)   (what bn_bwd_apply_kernel consumes)
  float* bwd_dgamma;              // [C] out: sum(dz * xhat)
  float* bwd_dbeta;               // [C] out: sum(dz)
};

// shared-memory bytes the epilogue needs: staging tile + statistics accumulators
__host__ __device__ constexpr int staging_bytes(int block_n) { return block_n * 128 * 2; }          // 128 rows x block_n bf16
__host__ __device__ constexpr int stat_bytes() { return 4 * 2 * STAT_MAX_C * 4; }                   // [4 warps][2][512] fp32

// Drain one accumulator tile.  Called by all 128 threads of the MMA warpgroup (et = 0..127), straight from the wgmma fragment:
// each thread takes its own column pairs of four tile rows (tc::frag_row / tc::frag_col) and writes them as bf16x2 words into the
// staging tile.  For a fixed (h, j, rr) the 32 lanes of a warp cover 8 rows x 4 words of 16-byte chunk j ^ (row & 7): 32 distinct
// banks, no conflicts, and no shared-memory round trip or barrier between the accumulators and the staged tile.
//   acc       : the tile's accumulators (wgmma fragment of this thread)
//   sbuf      : staging tile (1024-byte aligned), valid_rows: rows of the tile that are real pixels (partial batch tiles)
//   col0, Cn  : first output channel of the tile, output channels
//   resid     : optional tensor of the output's shape added to the tile before rounding (dgrad: the gradient arriving over the
//               other branch of a fork, e.g. the residual shortcut)
//   mask      : optional tensor of the output's shape; the output is zeroed where it is <= 0 (ReLU backward of the BatchNorm output
//               that fed this convolution), after the residual add
//   row_off(r): element offset of channel 0 of tile row r in those tensors (only called for r < valid_rows)
// Per element: acc (+ bias) (+ resid) (mask), rounded once to nearest even -- the staged tile is what the TMA store and the
// statistics read.
template <int BLOCK_N, typename RowOff>
__device__ __forceinline__ void drain_tile(const float (&acc)[2][BLOCK_N / 2], uint8_t* sbuf, int et, int valid_rows, int col0, int Cn,
                                           const float* bias_f32, const __nv_bfloat16* bias_bf16, const __nv_bfloat16* resid,
                                           const __nv_bfloat16* mask, RowOff row_off) {
  const int cols = Cn - col0;                      // 64-column box b of the tile is real iff 64 b < cols (Cn % 64 == 0)
  const int cq = tc::frag_col(et, 0);              // this thread's first column inside a block
  // the previous tile's TMA store (and every thread's statistics pass) must have finished READING the staging tile
  if (et == 0) tc::tma_store_wait_read<0>();
  tc::named_bar_sync(EPI_BAR_ID, EPI_THREADS);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int r = tc::frag_row(et, h, rr);
      const uint32_t srow = tc::smem_u32(sbuf) + r * 128 + 4 * (et & 3);
      // one 64-column box at a time: at most 8 column pairs and 8 residual / mask words in flight (register pressure)
#pragma unroll
      for (int box = 0; box < BLOCK_N / 64; ++box) {
        if (64 * box >= cols) continue;            // Cn % 64 == 0: the box is real or entirely beyond Cn
        float v[8][2];
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          v[jj][0] = acc[h][4 * (8 * box + jj) + 2 * rr];
          v[jj][1] = acc[h][4 * (8 * box + jj) + 2 * rr + 1];
        }
        const int cc0 = col0 + 64 * box + cq;
        if (bias_f32 || bias_bf16) {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int cc = cc0 + 8 * jj;
            v[jj][0] += bias_f32 ? bias_f32[cc] : __bfloat162float(bias_bf16[cc]);
            v[jj][1] += bias_f32 ? bias_f32[cc + 1] : __bfloat162float(bias_bf16[cc + 1]);
          }
        }
        if ((resid || mask) && r < valid_rows) {
          const long long off = row_off(r) + cc0;
          __nv_bfloat162 g[8];
          if (resid) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) g[jj] = __ldg(reinterpret_cast<const __nv_bfloat162*>(resid + off + 8 * jj));
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) { const float2 f = __bfloat1622float2(g[jj]); v[jj][0] += f.x; v[jj][1] += f.y; }
          }
          if (mask) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) g[jj] = __ldg(reinterpret_cast<const __nv_bfloat162*>(mask + off + 8 * jj));
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const float2 f = __bfloat1622float2(g[jj]);
              v[jj][0] = f.x > 0.f ? v[jj][0] : 0.f;
              v[jj][1] = f.y > 0.f ? v[jj][1] : 0.f;
            }
          }
        }
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)                 // ordered before the fence below: both volatile
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(srow + box * (128 * 128) + ((jj ^ (r & 7)) << 4)), "r"(tc::pack2(v[jj][0], v[jj][1])));
      }
    }
  }
  tc::fence_async_smem();                          // generic-proxy writes -> visible to the TMA store
  tc::named_bar_sync(EPI_BAR_ID, EPI_THREADS);
}

// Per-channel sum / sum of squares of the staged (bf16-rounded) tiles, kept in REGISTERS across the tiles of a CTA: epilogue
// thread et owns the 16-byte chunk (8 channels) j = et & 7 of every 64-channel half and the rows rg, rg + 16, ... (rg = et >> 3),
// i.e. eight 16-byte shared-memory loads per half per tile (conflict-free: a quarter warp reads one 128-byte row).
template <int BLOCK_N>
struct StatAcc {
  float s[BLOCK_N / 8], q[BLOCK_N / 8];
  __device__ __forceinline__ void clear() {
#pragma unroll
    for (int i = 0; i < BLOCK_N / 8; ++i) { s[i] = 0.f; q[i] = 0.f; }
  }
  __device__ __forceinline__ void add_tile(const uint8_t* sbuf, int et, int valid_rows) {
    const int j = et & 7, rg = et >> 3;
#pragma unroll
    for (int box = 0; box < BLOCK_N / 64; ++box) {
      const uint8_t* base = sbuf + box * (128 * 128);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = rg + 16 * i;
        if (r < valid_rows) {
          const uint4 v = *reinterpret_cast<const uint4*>(base + r * 128 + ((j ^ (r & 7)) << 4));
          const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 f = __bfloat1622float2(p[e]);
            s[box * 8 + 2 * e] += f.x;          q[box * 8 + 2 * e] = fmaf(f.x, f.x, q[box * 8 + 2 * e]);
            s[box * 8 + 2 * e + 1] += f.y;      q[box * 8 + 2 * e + 1] = fmaf(f.y, f.y, q[box * 8 + 2 * e + 1]);
          }
        }
      }
    }
  }
  // BatchNorm-backward flavour: s += dz, q += dz * xhat with xhat = (x - mean) * invstd; dz is the staged (rounded, masked) tile,
  // x is read from global memory -- row r of the tile lives at x + row_off(r) (channel 0 of that pixel), columns col0 + ...
  template <typename RowOff>
  __device__ __forceinline__ void add_tile_bwd(const uint8_t* sbuf, int et, int valid_rows, const __nv_bfloat16* x, RowOff row_off,
                                               int col0, int Cn, const float* mean, const float* invstd) {
    const int j = et & 7, rg = et >> 3;
#pragma unroll
    for (int box = 0; box < BLOCK_N / 64; ++box) {
      const int cbase = col0 + box * 64 + j * 8;
      if (cbase >= Cn) continue;
      float mu[8], is[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) { mu[e] = __ldg(mean + cbase + e); is[e] = __ldg(invstd + cbase + e); }
      const uint8_t* base = sbuf + box * (128 * 128);
      uint4 xv[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = rg + 16 * i;
        if (r < valid_rows) xv[i] = __ldg(reinterpret_cast<const uint4*>(x + row_off(r) + cbase));
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = rg + 16 * i;
        if (r < valid_rows) {
          const uint4 v = *reinterpret_cast<const uint4*>(base + r * 128 + ((j ^ (r & 7)) << 4));
          const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
          const __nv_bfloat162* px = reinterpret_cast<const __nv_bfloat162*>(&xv[i]);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 d = __bfloat1622float2(p[e]);
            const float2 xx = __bfloat1622float2(px[e]);
            s[box * 8 + 2 * e] += d.x;
            q[box * 8 + 2 * e] = fmaf(d.x, (xx.x - mu[2 * e]) * is[2 * e], q[box * 8 + 2 * e]);
            s[box * 8 + 2 * e + 1] += d.y;
            q[box * 8 + 2 * e + 1] = fmaf(d.y, (xx.y - mu[2 * e + 1]) * is[2 * e + 1], q[box * 8 + 2 * e + 1]);
          }
        }
      }
    }
  }
  // fold the four row groups of a warp (fixed xor tree) and add to this warp's shared-memory accumulators [warp][2][C]
  __device__ __forceinline__ void flush(float* s_stat, int et, int col0, int Cn) {
    const int j = et & 7, warp = et >> 5;
#pragma unroll
    for (int i = 0; i < BLOCK_N / 8; ++i) {
      float a = s[i], b = q[i];
      a += __shfl_xor_sync(0xffffffffu, a, 8);  b += __shfl_xor_sync(0xffffffffu, b, 8);
      a += __shfl_xor_sync(0xffffffffu, a, 16); b += __shfl_xor_sync(0xffffffffu, b, 16);
      const int c = col0 + (i >> 3) * 64 + j * 8 + (i & 7);
      if ((et & 31) < 8 && c < Cn) {
        float* acc = s_stat + (warp * 2) * STAT_MAX_C + c;
        acc[0] += a;
        acc[STAT_MAX_C] += b;
      }
    }
    clear();
  }
};
constexpr int STAT_PARTS = 4;             // one accumulator row per epilogue warp

// Kernel tail, executed by ALL threads of the CTA after the role loops joined (__syncthreads before the call).
//   slot / nslots: workspace row of this CTA / number of rows the last CTA folds
//   c_lo, c_hi   : channel range this CTA writes into its slot (the others in the slot are written by sibling CTAs or are zero)
template <int NUM_THREADS>
__device__ __forceinline__ void finalize_stats(const BnStatArgs& st, float* s_stat, int parts, int Cn, int slot, int nslots,
                                               int c_lo, int c_hi, float* s_scratch /* >= NUM_THREADS * 4 floats */,
                                               int ticket = 0, int ticket_arrivals = -1) {
  // This CTA's partial sums of channels [c_lo, c_hi) go to slot `slot`; the LAST of the `ticket_arrivals` CTAs that share ticket
  // counter `ticket` (all CTAs of the grid, or the CTAs of one channel tile when every tile has its own CTA) folds the nslots
  // partials of those channels in a fixed order and publishes mean / invstd (+ running statistics).
  __shared__ int s_is_last;
  const int width = c_hi - c_lo;                   // multiple of 4
  for (int i = threadIdx.x; i < 2 * width; i += NUM_THREADS) {
    const int a = i / width, c = c_lo + i % width;
    float t = 0.f;
    for (int p = 0; p < parts; ++p) t += s_stat[(p * 2 + a) * STAT_MAX_C + c];
    st.partial[((long long)slot * 2 + a) * Cn + c] = t;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // release: the partial stores of the whole CTA (ordered before this thread by the barrier) become visible with the ticket;
    // acquire: the last CTA sees every other CTA's partials.  One acq_rel atomic instead of two gpu-scope fences around a relaxed one.
    unsigned int prev;
    unsigned int* ctr = st.counter + ticket;
    asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(prev) : "l"(ctr) : "memory");
    const unsigned int last = (unsigned int)(ticket_arrivals < 0 ? (int)gridDim.x : ticket_arrivals) - 1u;
    s_is_last = (prev == last);
    if (s_is_last) *ctr = 0;
  }
  __syncthreads();
  if (!s_is_last) return;
  // fold: items4 = 2 * width / 4 float4 columns, SUB interleaved subsets of the slots; fixed order everywhere
  const int w4 = width >> 2;
  const int items4 = 2 * w4;
  const int SUB = NUM_THREADS / items4 > 0 ? NUM_THREADS / items4 : 1;
  for (int i0 = 0; i0 < items4; i0 += NUM_THREADS) {                 // one pass unless 2 * width / 4 > NUM_THREADS
    const int item = i0 + (int)threadIdx.x % (items4 < NUM_THREADS ? items4 : NUM_THREADS);
    const int sub = items4 < NUM_THREADS ? (int)threadIdx.x / items4 : 0;
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    if (sub < SUB && item < items4) {
      const int a = item / w4, c4 = item - a * w4;
      const float* col = st.partial + (long long)a * Cn + c_lo + c4 * 4;          // + slot * 2 * Cn
      constexpr int FB = 32;                                          // independent 16-byte loads in flight
      for (int g0 = sub; g0 < nslots; g0 += FB * SUB) {
        float4 v[FB];
#pragma unroll
        for (int u = 0; u < FB; ++u) {
          const int g = g0 + u * SUB;
          v[u] = g < nslots ? __ldcg(reinterpret_cast<const float4*>(col + (long long)g * 2 * Cn)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < FB; ++u) { t.x += v[u].x; t.y += v[u].y; t.z += v[u].z; t.w += v[u].w; }      // fixed order
      }
    }
    __syncthreads();
    reinterpret_cast<float4*>(s_scratch)[threadIdx.x] = t;
    __syncthreads();
    // subset 0 combines the subsets in order and leaves the totals in s_stat: [2][width], a-major
    if (sub == 0 && item < items4) {
      float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
      const int nsub = items4 < NUM_THREADS ? SUB : 1;
      for (int s2 = 0; s2 < nsub; ++s2) {
        const float4 v = reinterpret_cast<const float4*>(s_scratch)[s2 * items4 + (item - i0)];
        tot.x += v.x; tot.y += v.y; tot.z += v.z; tot.w += v.w;
      }
      reinterpret_cast<float4*>(s_stat)[item] = tot;
    }
  }
  __syncthreads();
  const float inv_m = 1.0f / (float)st.count;
  if (st.bwd_x) {                                  // BatchNorm-backward mode: totals are sum(dz), sum(dz * xhat)
    for (int i = threadIdx.x; i < width; i += NUM_THREADS) {
      const int c = c_lo + i;
      const float sd = s_stat[i], sq = s_stat[width + i];
      st.bwd_dbeta[c] = sd;
      st.bwd_dgamma[c] = sq;
      st.bwd_sums[c] = sd * inv_m;
      st.bwd_sums[Cn + c] = sq * inv_m;
    }
    return;
  }
  for (int i = threadIdx.x; i < width; i += NUM_THREADS) {
    const int c = c_lo + i;
    const float m = s_stat[i] * inv_m;
    float var = fmaf(-m, m, s_stat[width + i] * inv_m);
    var = var < 0.f ? 0.f : var;
    st.mean[c] = m;
    st.invstd[c] = rsqrtf(var + st.eps);
    if (st.running_mean) {
      // __fmul_rn: rounded on its own, never contracted into the fma below (bn_fused.cu's finalisation does the same, so the
      // epilogue and the standalone statistics kernel update the running variance bit-identically)
      const float unbiased = st.count > 1 ? __fmul_rn(var, (float)st.count / (float)(st.count - 1)) : var;
      st.running_mean[c] = fmaf(st.momentum, m - st.running_mean[c], st.running_mean[c]);
      st.running_var[c] = fmaf(st.momentum, unbiased - st.running_var[c], st.running_var[c]);
    }
  }
}

}  // namespace convepi
