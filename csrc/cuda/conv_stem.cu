// K10 (convolution part, continued): the 3-channel stem convolution (3x3 / stride 1 / pad 1, Cin = 3, Cout = 64) on CUDA cores.
//
// K = 27 is far too small for the tensor-core path (a wgmma K-step is 16 and a TMA row must be a multiple of 16 bytes; a
// 3-channel bf16 pixel is 6 bytes), and the work is tiny: 0.45 GFLOP per ResNet-18 step at B = 128, but the output / dy
// tensors are the largest of the network (16.8 MB).  Pairing every FMA with a shared-memory load makes such a kernel slow, hence this layout:
//
//   stem_fprop_kernel : persistent CTAs over 256-pixel tiles.  The (rows+2) x (W+2) input halo patch sits in shared memory as
//                       fp32 float4 per pixel (3 channels + pad), the 27 x 64 weights as fp32.  A thread computes 4 consecutive
//                       pixels x 16 output channels: one 16-byte weight load feeds 16 FMAs, one 16-byte patch load 48.  The four
//                       threads of a pixel write 128 contiguous bytes.  Optionally the kernel also produces the training-mode
//                       BatchNorm statistics of its (bf16-rounded) output: per-thread sums over all tiles of the CTA, one
//                       fixed-order fold per CTA, last-CTA fold of the per-CTA partials (conv_epilogue.cuh).
//   stem_wgrad_kernel : persistent CTAs over the same tiles; dy tile [256][64] bf16 and the x patch in shared memory.  Thread
//                       (pixel subset, 4 output channels) keeps all 27 x 4 filter-gradient entries in registers: per pixel one
//                       8-byte dy load + nine 16-byte patch loads feed 108 FMAs.  One fixed-order cross-subset fold per CTA,
//                       then stem_wgrad_reduce_kernel folds the per-CTA partials (8 interleaved subsets per output element).
//   (no dgrad: the network input needs no gradient)
//
// Bit-determinism: tile -> CTA assignment and every summation order depend only on the shape and the grid size.
//
// Reference counterpart: `self.conv1 = nn.Conv2d(3, 64, kernel_size=3, stride=1, padding=1, bias=False)` of
// src/model_ops/resnet.py:70-72 and the first layer of src/model_ops/vgg.py:46-59 (PyTorch-0.3 CPU THNN).
#include "conv_epilogue.cuh"

namespace {

constexpr int CIN = 3;
constexpr int KTOT = 27;            // 3 x 3 x 3, index k = (r*3 + s)*3 + ci  (the arena layout of a [Cout,3,3,3] weight row)
constexpr int COUT = 64;
constexpr int TILE_PX = 256;
constexpr int THREADS = 256;
constexpr int MAX_PATCH_PX = 400;   // max over W in {8,16,32,64} of (256/W + 2) * (W + 2) = 396 (W = 64)
constexpr int FPROP_SX = 1024;      // fprop reuses the patch buffer as [64][64] fp32 fold scratch

struct StemArgs {
  const __nv_bfloat16* x;          // [N, H, W, 3]
  const __nv_bfloat16* w;          // [64, 3, 3, 3]
  __nv_bfloat16* y;                // [N, H, W, 64]
  const float* bias;               // [64] or null
  int N, H, W;
  int rows_per_tile;               // rows_per_tile * W == 256
  int tiles;                       // N * H / rows_per_tile
  convepi::BnStatArgs stat;
};

// x halo patch of a tile as float4 per pixel (ci 0..2, pad), zero outside the image
__device__ __forceinline__ void load_patch(float4* sx, const __nv_bfloat16* x, int n, int h0, int H, int W, int RT) {
  const int PWD = W + 2;
  for (int i = threadIdx.x; i < (RT + 2) * PWD; i += THREADS) {
    const int col = i % PWD - 1, row = i / PWD - 1 + h0;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row >= 0 && row < H && col >= 0 && col < W) {
      const __nv_bfloat16* p = x + (((long long)n * H + row) * W + col) * CIN;
      v.x = __bfloat162float(p[0]); v.y = __bfloat162float(p[1]); v.z = __bfloat162float(p[2]);
    }
    sx[i] = v;
  }
}

__global__ void __launch_bounds__(THREADS) stem_fprop_kernel(const StemArgs a) {
  __shared__ __align__(16) float ws[KTOT][COUT];                              // 6.9 KB
  __shared__ __align__(16) float4 sx[FPROP_SX];                               // 16 KB
  __shared__ __align__(16) float s_red[2 * convepi::STAT_MAX_C + 4 * THREADS]; // statistics: totals + fold scratch
  for (int i = threadIdx.x; i < KTOT * COUT; i += THREADS) {
    const int co = i / KTOT, k = i - co * KTOT;
    ws[k][co] = __bfloat162float(a.w[i]);
  }
  const int W = a.W, RT = a.rows_per_tile, PWD = W + 2;
  const int cg = threadIdx.x & 3, pg = threadIdx.x >> 2;                      // 16-channel group, 4-pixel group
  const int gpr = W >> 2;                                                      // pixel groups per image row
  const int prow = pg / gpr, pcol = (pg % gpr) * 4;
  const bool want_stats = a.stat.partial != nullptr;
  float st_s[16], st_q[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) { st_s[j] = 0.f; st_q[j] = 0.f; }
  const int tiles_per_img = a.H / RT;

  for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
    const int n = tile / tiles_per_img, h0 = (tile - n * tiles_per_img) * RT;
    __syncthreads();                                                          // previous tile's patch no longer read (and ws ready)
    load_patch(sx, a.x, n, h0, a.H, W, RT);
    __syncthreads();
    float acc[4][16];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[p][j] = a.bias ? a.bias[cg * 16 + j] : 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      float4 in[6];
#pragma unroll
      for (int c = 0; c < 6; ++c) in[c] = sx[(prow + r) * PWD + pcol + c];
#pragma unroll
      for (int s = 0; s < 3; ++s) {
#pragma unroll
        for (int ci = 0; ci < 3; ++ci) {
          const int k = (r * 3 + s) * 3 + ci;
          const float4* wr = reinterpret_cast<const float4*>(&ws[k][cg * 16]);
          const float4 w0 = wr[0], w1 = wr[1], w2 = wr[2], w3 = wr[3];
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            const float4 iv = in[p + s];
            const float v = ci == 0 ? iv.x : (ci == 1 ? iv.y : iv.z);
            acc[p][0] = fmaf(v, w0.x, acc[p][0]);   acc[p][1] = fmaf(v, w0.y, acc[p][1]);
            acc[p][2] = fmaf(v, w0.z, acc[p][2]);   acc[p][3] = fmaf(v, w0.w, acc[p][3]);
            acc[p][4] = fmaf(v, w1.x, acc[p][4]);   acc[p][5] = fmaf(v, w1.y, acc[p][5]);
            acc[p][6] = fmaf(v, w1.z, acc[p][6]);   acc[p][7] = fmaf(v, w1.w, acc[p][7]);
            acc[p][8] = fmaf(v, w2.x, acc[p][8]);   acc[p][9] = fmaf(v, w2.y, acc[p][9]);
            acc[p][10] = fmaf(v, w2.z, acc[p][10]); acc[p][11] = fmaf(v, w2.w, acc[p][11]);
            acc[p][12] = fmaf(v, w3.x, acc[p][12]); acc[p][13] = fmaf(v, w3.y, acc[p][13]);
            acc[p][14] = fmaf(v, w3.z, acc[p][14]); acc[p][15] = fmaf(v, w3.w, acc[p][15]);
          }
        }
      }
    }
    __nv_bfloat16* orow = a.y + ((((long long)n * a.H + h0 + prow) * W + pcol) * COUT) + cg * 16;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const uint4 lo = tc::pack8(&acc[p][0]), hi = tc::pack8(&acc[p][8]);
      uint4* dst = reinterpret_cast<uint4*>(orow + p * COUT);
      dst[0] = lo; dst[1] = hi;
      if (want_stats) {
        const __nv_bfloat162* b0 = reinterpret_cast<const __nv_bfloat162*>(&lo);
        const __nv_bfloat162* b1 = reinterpret_cast<const __nv_bfloat162*>(&hi);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 u = __bfloat1622float2(b0[j]), v = __bfloat1622float2(b1[j]);
          st_s[2 * j] += u.x; st_q[2 * j] = fmaf(u.x, u.x, st_q[2 * j]);
          st_s[2 * j + 1] += u.y; st_q[2 * j + 1] = fmaf(u.y, u.y, st_q[2 * j + 1]);
          st_s[8 + 2 * j] += v.x; st_q[8 + 2 * j] = fmaf(v.x, v.x, st_q[8 + 2 * j]);
          st_s[8 + 2 * j + 1] += v.y; st_q[8 + 2 * j + 1] = fmaf(v.y, v.y, st_q[8 + 2 * j + 1]);
        }
      }
    }
  }
  if (!want_stats) return;
  // CTA fold over the 64 pixel groups (fixed order): scratch [64 pg][64 co] per statistic, staged through the patch buffer
  float* scratch = reinterpret_cast<float*>(sx);                               // 64 * 64 floats = 16 KB
#pragma unroll 1
  for (int which = 0; which < 2; ++which) {
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 16; ++j) scratch[pg * COUT + cg * 16 + j] = which ? st_q[j] : st_s[j];
    __syncthreads();
    if (threadIdx.x < COUT) {
      float t0 = 0.f, t1 = 0.f;
      for (int g = 0; g < 64; g += 2) { t0 += scratch[g * COUT + threadIdx.x]; t1 += scratch[(g + 1) * COUT + threadIdx.x]; }
      s_red[which * convepi::STAT_MAX_C + threadIdx.x] = t0 + t1;
    }
  }
  __syncthreads();
  convepi::finalize_stats<THREADS>(a.stat, s_red, 1, COUT, (int)blockIdx.x, (int)gridDim.x, 0, COUT, s_red + 2 * convepi::STAT_MAX_C);
}

struct StemWgradArgs {
  const __nv_bfloat16* dy;         // [N, H, W, 64]
  const __nv_bfloat16* x;          // [N, H, W, 3]
  float* partial;                  // [grid][64][27]
  int N, H, W;
  int rows_per_tile;               // rows_per_tile * W == 256
  int tiles;                       // N * H / rows_per_tile
};

__global__ void __launch_bounds__(THREADS) stem_wgrad_kernel(const StemWgradArgs a) {
  __shared__ __align__(16) __nv_bfloat16 sdy[TILE_PX * COUT];                 // 32 KB (reused for the final fold)
  __shared__ __align__(16) float4 sx[MAX_PATCH_PX];
  const int cq = threadIdx.x & 15, ps = threadIdx.x >> 4;                     // 4-output-channel group, pixel subset (16 pixels / tile)
  const int W = a.W, RT = a.rows_per_tile, PWD = W + 2;
  float acc[4][KTOT];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int k = 0; k < KTOT; ++k) acc[c][k] = 0.f;
  const int tiles_per_img = a.H / RT;

  for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
    const int n = tile / tiles_per_img, h0 = (tile - n * tiles_per_img) * RT;
    __syncthreads();                                                          // previous tile's smem no longer read
    {
      const uint4* src = reinterpret_cast<const uint4*>(a.dy + (((long long)n * a.H + h0) * W) * COUT);
      uint4* dst = reinterpret_cast<uint4*>(sdy);
#pragma unroll
      for (int i = 0; i < TILE_PX * COUT / 8 / THREADS; ++i) dst[threadIdx.x + i * THREADS] = src[threadIdx.x + i * THREADS];
    }
    load_patch(sx, a.x, n, h0, a.H, W, RT);
    __syncthreads();
#pragma unroll 2
    for (int i = 0; i < TILE_PX / 16; ++i) {
      const int px = ps + i * 16;
      const uint2 dv = *reinterpret_cast<const uint2*>(sdy + px * COUT + cq * 4);
      const float2 d01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&dv.x));
      const float2 d23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&dv.y));
      const float d[4] = {d01.x, d01.y, d23.x, d23.y};
      const int base = (px / W) * PWD + (px % W);                              // patch index of the (r = 0, s = 0) neighbour
#pragma unroll
      for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const float4 xv = sx[base + r * PWD + s];
          const int k = (r * 3 + s) * 3;
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            acc[c][k] = fmaf(d[c], xv.x, acc[c][k]);
            acc[c][k + 1] = fmaf(d[c], xv.y, acc[c][k + 1]);
            acc[c][k + 2] = fmaf(d[c], xv.z, acc[c][k + 2]);
          }
        }
      }
    }
  }
  // fold the 16 pixel subsets in a fixed order, one output channel of each thread's four per pass (27.6 KB of scratch)
  float* red = reinterpret_cast<float*>(sdy);                                  // [16 ps][16 cq][27]
  float* out = a.partial + (long long)blockIdx.x * COUT * KTOT;
#pragma unroll 1
  for (int c = 0; c < 4; ++c) {
    __syncthreads();
#pragma unroll
    for (int k = 0; k < KTOT; ++k) {
      float v = acc[0][k];
      if (c == 1) v = acc[1][k]; else if (c == 2) v = acc[2][k]; else if (c == 3) v = acc[3][k];
      red[(ps * 16 + cq) * KTOT + k] = v;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 16 * KTOT; i += THREADS) {                   // i = cq' * 27 + k
      float t0 = 0.f, t1 = 0.f;
      for (int p = 0; p < 16; p += 2) { t0 += red[p * 16 * KTOT + i]; t1 += red[(p + 1) * 16 * KTOT + i]; }
      const int cq2 = i / KTOT, k = i - cq2 * KTOT;
      out[(cq2 * 4 + c) * KTOT + k] = t0 + t1;
    }
  }
}

// out element e (of 64 * 27): 8 interleaved subsets of the per-CTA partials, combined in a fixed order
__global__ void __launch_bounds__(256) stem_wgrad_reduce_kernel(const float* partial, int parts, __nv_bfloat16* dw) {
  __shared__ float s[8][32];
  const int il = threadIdx.x & 31, sub = threadIdx.x >> 5;
  const int e = blockIdx.x * 32 + il;
  float t0 = 0.f, t1 = 0.f;
  if (e < COUT * KTOT) {
    int p = sub;
    for (; p + 8 < parts; p += 16) { t0 += partial[(long long)p * COUT * KTOT + e]; t1 += partial[(long long)(p + 8) * COUT * KTOT + e]; }
    if (p < parts) t0 += partial[(long long)p * COUT * KTOT + e];
  }
  s[sub][il] = t0 + t1;
  __syncthreads();
  if (sub == 0 && e < COUT * KTOT) {
    float t = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) t += s[q][il];
    dw[e] = __float2bfloat16_rn(t);
  }
}

bool pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

int stem_grid(int tiles, int num_sms) { return tiles < 2 * num_sms ? tiles : 2 * num_sms; }

}  // namespace

extern "C" int drc_conv_stem_supported(int H, int W, int Cin, int Cout) {
  return Cin == 3 && Cout == 64 && pow2(W) && W >= 8 && W <= 64 && H % (TILE_PX / W) == 0;
}

// grid of the stem kernels (= number of fp32 wgrad partials [64][27] and of statistics slots in the workspaces)
extern "C" int drc_conv_stem_wgrad_parts(int N, int H, int W, int num_sms) {
  return stem_grid(N * (H / (TILE_PX / W)), num_sms);
}

// stat_*: optional BatchNorm statistics of y (see drc_convg); workspace = drc_conv_stem_wgrad_parts(...) * 128 floats.
extern "C" int drc_conv_stem_fprop(const void* x, const void* w, void* y, const float* bias, int N, int H, int W, float* stat_partial,
                                   unsigned int* stat_counter, float* stat_mean, float* stat_invstd, float* running_mean,
                                   float* running_var, float eps, float momentum, int num_sms, int device, cudaStream_t stream) {
  if (!drc_conv_stem_supported(H, W, 3, 64)) return -1;
  if (device >= 0) { cudaError_t e = cudaSetDevice(device); if (e != cudaSuccess) return (int)e; }
  StemArgs a;
  a.x = (const __nv_bfloat16*)x; a.w = (const __nv_bfloat16*)w; a.y = (__nv_bfloat16*)y; a.bias = bias;
  a.N = N; a.H = H; a.W = W; a.rows_per_tile = TILE_PX / W; a.tiles = N * (H / a.rows_per_tile);
  a.stat.partial = stat_partial; a.stat.counter = stat_counter; a.stat.mean = stat_mean; a.stat.invstd = stat_invstd;
  a.stat.running_mean = running_mean; a.stat.running_var = running_var; a.stat.count = (long long)N * H * W;
  a.stat.eps = eps; a.stat.momentum = momentum;
  a.stat.bwd_x = nullptr; a.stat.bwd_mask = nullptr;           // forward statistics only
  stem_fprop_kernel<<<stem_grid(a.tiles, num_sms), THREADS, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

// ws: fp32 workspace of drc_conv_stem_wgrad_parts(...) * 64 * 27 elements; dw: [64,3,3,3] bf16.
extern "C" int drc_conv_stem_wgrad(const void* dy, const void* x, void* dw, float* ws, int N, int H, int W, int num_sms, int device,
                                   cudaStream_t stream) {
  if (!drc_conv_stem_supported(H, W, 3, 64)) return -1;
  if (device >= 0) { cudaError_t e = cudaSetDevice(device); if (e != cudaSuccess) return (int)e; }
  StemWgradArgs a;
  a.dy = (const __nv_bfloat16*)dy; a.x = (const __nv_bfloat16*)x; a.partial = ws;
  a.N = N; a.H = H; a.W = W; a.rows_per_tile = TILE_PX / W; a.tiles = N * (H / a.rows_per_tile);
  const int parts = stem_grid(a.tiles, num_sms);
  stem_wgrad_kernel<<<parts, THREADS, 0, stream>>>(a);
  int rc = (int)cudaGetLastError();
  if (rc) return rc;
  stem_wgrad_reduce_kernel<<<(COUT * KTOT + 31) / 32, 256, 0, stream>>>(ws, parts, (__nv_bfloat16*)dw);
  return (int)cudaGetLastError();
}
