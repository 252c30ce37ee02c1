// K10 (convolution part, continued): HALO-REUSE 3x3 / stride-1 convolution on wgmma for the 64 -> 64 channel layers.
//
// On the layer1 shape (128 x 64 x 32 x 32) a per-tap kernel (conv_tap_wgmma.cu) is bound by L2 -> SM traffic: every filter tap
// re-loads the shifted activation patch and its 8 KB weight slice for every tile.  With Cin = Cout = 64 everything a CTA needs
// fits in shared memory:
//
//   * the nine weight taps (9 x 8 KB) are loaded ONCE per CTA and stay resident (the CTA is persistent over tiles);
//   * an M tile is an 8 x 16 pixel block; its halo is loaded ONCE per tile as three column-shifted boxes of (16+2) rows x 8
//     pixels (box s holds input columns w0 - 1 + s .. w0 + 6 + s; out-of-image pixels zero-filled), 54 KB instead of the 9 x 16 KB
//     a per-tap kernel streams;
//   * the A operand of tap (r, s) is box s from image row r on: a dense 128-row K-major tile that starts r * 1024 bytes into the
//     box, i.e. on a swizzle-pattern boundary, so the wgmma descriptor needs no base offset.
//
// dgrad is the same kernel with mirrored taps and the weight tile read MN-major (same shared-memory image).
// The epilogue is the shared staged TMA-store epilogue of conv_epilogue.cuh, including the fused BatchNorm statistics.
//
// Reference counterpart: the 64 -> 64 BasicBlock convolutions of src/model_ops/resnet.py:14-36.
#include "conv_epilogue.cuh"
#include "wgmma_common.cuh"

namespace {

using namespace tc;

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 64;          // Cout (fprop) / Cin (dgrad)
constexpr int NUM_THREADS = 256;
constexpr int TW = 8, TH = 16;       // tile = 8 x 16 pixels
constexpr int PH = TH + 2;           // halo rows
constexpr int BOX_BYTES = PH * TW * 128;             // 18432: one column-shifted box [18 rows][8 px][64 ch]
constexpr int HALO_BYTES = 3 * BOX_BYTES;            // 55296 (1024-byte multiple)
constexpr int W_TAP_BYTES = BLOCK_N * 128;           // 8 KB
constexpr int W_BYTES = 9 * W_TAP_BYTES;             // 72 KB
constexpr int STAGES = 2;
constexpr int EPI_BYTES = convepi::staging_bytes(BLOCK_N) + convepi::stat_bytes();
constexpr int SMEM_BYTES = W_BYTES + STAGES * HALO_BYTES + EPI_BYTES + 1024 + 256;
static_assert(SMEM_BYTES <= 227 * 1024, "H100: 227 KB of shared memory per block");

struct HaloArgs {
  int N, H, W;
  const __nv_bfloat16* resid;     // optional [N,H,W,64] tensor added to the output in the epilogue (dgrad: the other branch's gradient)
  const float* bias_f32;
  const __nv_bfloat16* bias_bf16;
  convepi::BnStatArgs stat;
};

// the three column-shifted halo boxes of the tile at (w0, h0, n0)
__device__ __forceinline__ void load_halo(uint8_t* dst, const CUtensorMap* tmap_x, int w0, int h0, int n0, uint64_t* bar) {
#pragma unroll
  for (int s = 0; s < 3; ++s) tma_load_4d(dst + s * BOX_BYTES, tmap_x, 0, w0 - 1 + s, h0 - 1, n0, bar);
}

template <bool DGRAD>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_halo_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                       const __grid_constant__ CUtensorMap tmap_out, const HaloArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_w = smem;                              // 9 taps x [64 rows][128 B]
  uint8_t* s_halo = smem + W_BYTES;                 // STAGES x HALO_BYTES
  uint8_t* sbuf = s_halo + STAGES * HALO_BYTES;     // staging tile [128][128 B]
  float* s_stat = reinterpret_cast<float*>(sbuf + convepi::staging_bytes(BLOCK_N));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sbuf + EPI_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* w_bar = empty_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wt = a.W / TW, ht = a.H / TH;
  const int num_tiles = wt * ht * a.N;
  const bool want_stats = a.stat.partial != nullptr;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmap_x);
    prefetch_tmap(&tmap_w);
    prefetch_tmap(&tmap_out);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }
    mbar_init(w_bar, 1);
    mbar_fence_init();
  }
  if (warp >= 4) {
    for (int i = threadIdx.x - 128; i < 2 * convepi::STAT_PARTS * convepi::STAT_MAX_C; i += convepi::EPI_THREADS) s_stat[i] = 0.f;
  }
  __syncthreads();

  if (warp == 0) {
    // ===================== TMA producer: weights once, then one halo per tile =====================
    if (elect_one()) {
      mbar_expect_tx(w_bar, W_BYTES);
      for (int tap = 0; tap < 9; ++tap) tma_load_2d(s_w + tap * W_TAP_BYTES, &tmap_w, tap * 64, 0, w_bar);
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int w0 = (tile % wt) * TW, h0 = ((tile / wt) % ht) * TH, n0 = tile / (wt * ht);
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_expect_tx(&full_bar[stage], (uint32_t)HALO_BYTES);
        load_halo(s_halo + stage * HALO_BYTES, &tmap_x, w0, h0, n0, &full_bar[stage]);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ===================== MMA (9 taps x 4 K-steps on one resident halo) + epilogue =====================
    const int et = threadIdx.x - 128;
    int stage = 0; uint32_t phase = 0;
    float acc[2][BLOCK_N / 2];
    convepi::StatAcc<BLOCK_N> sacc;
    sacc.clear();
    mbar_wait(w_bar, 0);
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int w0 = (tile % wt) * TW, h0 = ((tile / wt) % ht) * TH, n0 = tile / (wt * ht);
      if (want_stats && a.stat.bwd_x) {            // BatchNorm-backward mode: this tile's rows of x / y into L2 under the MMAs
        const long long off = (((long long)n0 * a.H + (h0 + et / TW)) * a.W + (w0 + et % TW)) * BLOCK_N;
        asm volatile("prefetch.global.L2 [%0];" ::"l"(a.stat.bwd_x + off));
        if (a.stat.bwd_mask) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.stat.bwd_mask + off));
      }
      mbar_wait(&full_bar[stage], phase);
      const uint32_t halo = smem_u32(s_halo + stage * HALO_BYTES);
      acc_undef<BLOCK_N / 2>(acc[0]);               // the previous tile's values: dead during its epilogue
      acc_undef<BLOCK_N / 2>(acc[1]);
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const int r = tap / 3, s = tap - 3 * r;
        // fprop: input pixel (y + r - 1, x + s - 1) = box s, row y + r; dgrad: (y + 1 - r, x + 1 - s) -> box 2 - s, row y + 2 - r
        const int pr = DGRAD ? 2 - r : r, ps = DGRAD ? 2 - s : s;
        // weights: K-major rows = Cout (fprop) or MN-major rows = Cout = K (dgrad)
        mma_kblock<BLOCK_N, false, DGRAD>(acc, halo + (uint32_t)(ps * BOX_BYTES + pr * 1024), smem_u32(s_w + tap * W_TAP_BYTES), tap == 0);
      }
      wgmma_wait<0>();
      fence_acc<BLOCK_N / 2>(acc[0]);
      fence_acc<BLOCK_N / 2>(acc[1]);
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
      auto row_off = [&](int r) -> long long { return (((long long)n0 * a.H + (h0 + r / TW)) * a.W + (w0 + r % TW)) * BLOCK_N; };
      convepi::drain_tile<BLOCK_N>(acc, sbuf, et, BLOCK_M, 0, BLOCK_N, a.bias_f32, a.bias_bf16, a.resid,
                                   want_stats ? a.stat.bwd_mask : nullptr, row_off);
      if (et == 0) {
        tma_store_4d(&tmap_out, sbuf, 0, w0, h0, n0);
        tma_store_commit();
      }
      if (want_stats) {
        if (a.stat.bwd_x) sacc.add_tile_bwd(sbuf, et, BLOCK_M, a.stat.bwd_x, row_off, 0, BLOCK_N, a.stat.bwd_mean, a.stat.bwd_invstd);
        else sacc.add_tile(sbuf, et, BLOCK_M);
      }
    }
    if (want_stats) sacc.flush(s_stat, et, 0, BLOCK_N);
    if (et == 0) tma_store_wait<0>();
  }

  __syncthreads();
  if (want_stats)
    convepi::finalize_stats<NUM_THREADS>(a.stat, s_stat, convepi::STAT_PARTS, BLOCK_N, (int)blockIdx.x, (int)gridDim.x, 0,
                                         BLOCK_N, reinterpret_cast<float*>(sbuf));
}

// ---------------------------------------------------------------------------------------------------------------------------
// Weight gradient of the same layers: dW[co][tap][ci] = sum_px dy[px][co] * x[px + tap][ci], ALL NINE TAPS FROM ONE RESIDENT HALO.
//
// Per 128-pixel tile: D_r[m = co][n = (s, ci)] += A[px][co] * B_r[px][(s, ci)]  with K = pixels, 16 per wgmma,
//   A   : the dy tile [128 px][64 co], MN-major (one 64-wide atom);
//   B_r : the three halo boxes of the forward kernel from image row r on, MN-major: N = 192 = taps (r, 0..2) x 64 ci -- the three
//         64-wide atoms are the three boxes, BOX_BYTES apart (the descriptor's leading-byte offset).
// Warpgroup g + 1 owns filter row r = g: a 64 x 192 fp32 accumulator (96 registers per thread) that lives across ALL tiles of the
// persistent CTA: one 70 KB TMA stage and 24 wgmmas per 128 pixels, no epilogue until the end.  Every CTA then writes one fp32
// partial [64][9][64] and wgrad_halo_reduce_kernel folds the per-CTA partials in a fixed order (bit-deterministic).
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int WG_THREADS = 512;                                   // producer warpgroup + three MMA warpgroups
constexpr int WG_DY_BYTES = BLOCK_M * 128;                        // 16 KB: [128 px][64 co]
constexpr int WG_STAGE = HALO_BYTES + WG_DY_BYTES;                // 70 KB
constexpr int WG_STAGES = 3;
constexpr int WG_SMEM = WG_STAGES * WG_STAGE + 1024 + 256;
static_assert(WG_SMEM <= 227 * 1024, "H100: 227 KB of shared memory per block");

struct HaloWgradArgs {
  int N, H, W;
  float* partial;                  // [grid][64 co][9 taps][64 ci]
};

__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad_halo_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_dy, const HaloWgradArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + WG_STAGES * WG_STAGE);
  uint64_t* empty_bar = full_bar + WG_STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wt = a.W / TW, ht = a.H / TH;
  const int num_tiles = wt * ht * a.N;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmap_x);
    prefetch_tmap(&tmap_dy);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < WG_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 12); }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (elect_one()) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int w0 = (tile % wt) * TW, h0 = ((tile / wt) % ht) * TH, n0 = tile / (wt * ht);
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sp = smem + stage * WG_STAGE;
        mbar_expect_tx(&full_bar[stage], (uint32_t)WG_STAGE);
        load_halo(sp, &tmap_x, w0, h0, n0, &full_bar[stage]);                           // x halo (zero-filled outside)
        tma_load_4d(sp + HALO_BYTES, &tmap_dy, 0, w0, h0, n0, &full_bar[stage]);         // dy tile
        if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    const int r = (warp >> 2) - 1;                                 // filter row of this warpgroup
    float acc[96];
    int stage = 0; uint32_t phase = 0;
    int prev = -1;
    bool first = true;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t halo = smem_u32(smem + stage * WG_STAGE);
      const uint32_t dyt = halo + HALO_BYTES;
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < BLOCK_M / MMA_K; ++ks) {                                     // 16 pixels = two image rows of the tile
        const uint64_t da = desc_mnmajor(dyt + ks * (MMA_K * 128), 64 * 128);
        const uint64_t db = desc_mnmajor(halo + (uint32_t)(r * 1024 + ks * (MMA_K * 128)), BOX_BYTES);
        Wgmma<192, 1, 1>::mma(acc, da, db, (first && ks == 0) ? 0u : 1u);
      }
      wgmma_commit();
      first = false;
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    fence_acc<96>(acc);
    // fragment -> fp32 partial: rows co = 16 w + l / 4 (+8), columns n = 8 j + 2 (l % 4) (+1) = (s, ci) of taps (r, 0..2)
    const int w = warp & 3;
    const int co = 16 * w + (lane >> 2);
    float* base = a.partial + (long long)blockIdx.x * (64 * 9 * 64) + (long long)co * (9 * 64) + r * 192 + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 24; ++j) {
      *reinterpret_cast<float2*>(base + 8 * j) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(base + 8 * (9 * 64) + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
}

// out[e] = sum over the per-CTA partials (8 interleaved subsets, each with up to 16 independent 16-byte loads in flight, combined
// in a fixed order), written as bf16.  elems = 64 * 9 * 64; grid = elems / 4 / 32 CTAs of 256 threads.
__global__ void __launch_bounds__(256) wgrad_halo_reduce_kernel(const float* partial, int parts, __nv_bfloat16* out) {
  constexpr int ELEMS4 = 64 * 9 * 64 / 4;
  __shared__ float4 s[8][32];
  const int il = threadIdx.x & 31, sub = threadIdx.x >> 5;
  const int e4 = blockIdx.x * 32 + il;
  const float4* p4 = reinterpret_cast<const float4*>(partial);
  float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int g0 = sub; g0 < parts; g0 += 8 * 16) {
    float4 v[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int g = g0 + 8 * u;
      v[u] = g < parts ? __ldcg(p4 + (long long)g * ELEMS4 + e4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) { t.x += v[u].x; t.y += v[u].y; t.z += v[u].z; t.w += v[u].w; }
  }
  s[sub][il] = t;
  __syncthreads();
  if (sub == 0) {
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < 8; ++k) { const float4 v = s[k][il]; r.x += v.x; r.y += v.y; r.z += v.z; r.w += v.w; }
    __nv_bfloat162 lo = __floats2bfloat162_rn(r.x, r.y), hi = __floats2bfloat162_rn(r.z, r.w);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&lo); o.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(out + (long long)e4 * 4) = o;
  }
}

}  // namespace

extern "C" int drc_conv_halo_supported(int H, int W, int Cin, int Cout) {
  return Cin == 64 && Cout == 64 && W % TW == 0 && H % TH == 0 && W >= TW && H >= TH;
}

extern "C" int drc_conv_halo_stat_slots(int N, int H, int W, int num_sms) {
  const int tiles = (W / TW) * (H / TH) * N;
  return tiles < num_sms ? tiles : num_sms;
}

// act: [N,H,W,64] bf16 (x for fprop, dy for dgrad); wgt: [64,3,3,64] bf16 (arena layout); out: [N,H,W,64] bf16.
// stat_*: optional fused BatchNorm statistics of the output (fprop only), see drc_convg.
extern "C" int drc_conv_halo(const void* act, const void* wgt, void* out, int N, int H, int W, int dgrad, const float* bias_f32,
                             const void* bias_bf16, const void* resid, float* stat_partial, unsigned int* stat_counter, float* stat_mean,
                             float* stat_invstd, float* running_mean, float* running_var, float eps, float momentum,
                             const void* bwd_x, const void* bwd_mask, const float* bwd_mean, const float* bwd_invstd, float* bwd_sums,
                             float* bwd_dgamma, float* bwd_dbeta, int num_sms, int device, cudaStream_t stream) {
  if (!drc_conv_halo_supported(H, W, 64, 64)) return -1;
  if (stat_partial && ((dgrad != 0) != (bwd_x != nullptr))) return -4;
  if (bwd_x && !(stat_partial && bwd_mean && bwd_invstd && bwd_sums && bwd_dgamma && bwd_dbeta)) return -7;
  if (device >= 0) { cudaError_t e = cudaSetDevice(device); if (e != cudaSuccess) return (int)e; }
  PFN_encodeTiled enc = get_encode();
  if (!enc) return -2;
  HaloArgs a;
  a.N = N; a.H = H; a.W = W; a.bias_f32 = bias_f32; a.bias_bf16 = (const __nv_bfloat16*)bias_bf16;
  a.resid = (const __nv_bfloat16*)resid;
  a.stat.partial = stat_partial; a.stat.counter = stat_counter; a.stat.mean = stat_mean; a.stat.invstd = stat_invstd;
  a.stat.running_mean = running_mean; a.stat.running_var = running_var; a.stat.count = (long long)N * H * W;
  a.stat.eps = eps; a.stat.momentum = momentum;
  a.stat.bwd_x = (const __nv_bfloat16*)bwd_x; a.stat.bwd_mask = (const __nv_bfloat16*)bwd_mask; a.stat.bwd_mean = bwd_mean;
  a.stat.bwd_invstd = bwd_invstd; a.stat.bwd_sums = bwd_sums; a.stat.bwd_dgamma = bwd_dgamma; a.stat.bwd_dbeta = bwd_dbeta;
  CUtensorMap tx, tw, tout;
  {
    cuuint64_t dims[4] = {64, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {128, (cuuint64_t)W * 128, (cuuint64_t)H * W * 128};
    cuuint32_t box[4] = {64, (cuuint32_t)TW, PH, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&tx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(act), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return 1000 + (int)r;
  }
  int r = encode_mat(&tw, wgt, 64, 9 * 64, 9 * 64, 64);
  if (r) return 2000 + r;
  r = encode_act(&tout, out, 64, W, H, N, TW, TH, 1, 1);
  if (r) return 3000 + r;
  const int tiles = (W / TW) * (H / TH) * N;
  const int grid = tiles < num_sms ? tiles : num_sms;
  static bool cfg0 = false, cfg1 = false;
  if (!dgrad) {
    auto kern = conv_halo_wgmma_kernel<false>;
    if (!cfg0) { cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES); if (e != cudaSuccess) return (int)e; cfg0 = true; }
    kern<<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(tx, tw, tout, a);
  } else {
    auto kern = conv_halo_wgmma_kernel<true>;
    if (!cfg1) { cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES); if (e != cudaSuccess) return (int)e; cfg1 = true; }
    kern<<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(tx, tw, tout, a);
  }
  return (int)cudaGetLastError();
}

// dy: [N,H,W,64] bf16, x: [N,H,W,64] bf16 -> dw: [64,3,3,64] bf16 (arena layout); ws: drc_conv_halo_stat_slots(...) * 36864 floats.
extern "C" int drc_conv_halo_wgrad(const void* dy, const void* x, void* dw, float* ws, int N, int H, int W, int num_sms, int device,
                                   cudaStream_t stream) {
  if (!drc_conv_halo_supported(H, W, 64, 64)) return -1;
  if (device >= 0) { cudaError_t e = cudaSetDevice(device); if (e != cudaSuccess) return (int)e; }
  PFN_encodeTiled enc = get_encode();
  if (!enc) return -2;
  CUtensorMap tx, tdy;
  {
    cuuint64_t dims[4] = {64, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {128, (cuuint64_t)W * 128, (cuuint64_t)H * W * 128};
    cuuint32_t box[4] = {64, (cuuint32_t)TW, PH, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&tx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(x), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return 1000 + (int)r;
  }
  int r = encode_act(&tdy, dy, 64, W, H, N, TW, TH, 1, 1);
  if (r) return 2000 + r;
  HaloWgradArgs a;
  a.N = N; a.H = H; a.W = W; a.partial = ws;
  const int grid = drc_conv_halo_stat_slots(N, H, W, num_sms);
  static bool cfgd = false;
  if (!cfgd) {
    cudaError_t e = cudaFuncSetAttribute(wgrad_halo_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM);
    if (e != cudaSuccess) return (int)e;
    cfgd = true;
  }
  wgrad_halo_wgmma_kernel<<<grid, WG_THREADS, WG_SMEM, stream>>>(tx, tdy, a);
  int rc = (int)cudaGetLastError();
  if (rc) return rc;
  wgrad_halo_reduce_kernel<<<64 * 9 * 64 / 4 / 32, 256, 0, stream>>>(ws, grid, (__nv_bfloat16*)dw);
  return (int)cudaGetLastError();
}
