// K10 (convolution part, continued): generalised tap-table implicit-GEMM convolutions on wgmma -- stride 1 or 2, 1x1 or 3x3.
//
// Machinery: TMA patch loads into 128B-swizzled tiles, wgmma 64xNx16 on both halves of a 128-pixel tile by one warpgroup with
// the accumulators in registers, epilogue from the accumulator fragments (wgmma_common.cuh).  What is specific is how a filter tap reaches the
// tensor core:
//
//   * strided fprop : the activation tensor map carries elementStrides {1, s, s, 1}, so ONE box load delivers the
//                     BW x BH x BN *output* pixels' inputs for a tap (every s-th pixel, halo zero-filled);
//   * strided dgrad : dx is split into its s x s parity classes; for class (ph, pw) only the taps with matching parity
//                     contribute and they read dy with unit stride -- 4 + 2 + 2 + 1 = 9 taps over the four classes of a
//                     3x3 / stride-2 layer (no zero-insertion, no wasted MMAs), all classes in ONE launch (class-major tile
//                     list, longest first); the epilogue writes with pixel stride s;
//   * strided wgrad : K-blocks are 64-pixel patches of dy; the matching x patch is a strided box shifted by the tap.
//
// A launch is described by a tap table (input offset + weight column per tap), so the stride-1 3x3 case is the
// 9-tap instance of the same kernel.  Motivation: the strided dgrads of ResNet-18 cost 5-10x their FLOP time in the library
// path (zero-insertion or one launch per parity class).
//
// The epilogue (conv_epilogue.cuh) stages the bf16 tile in swizzled shared memory straight from the accumulator fragments, stores
// it with ONE TMA tensor store per 64-channel half and can reduce it per channel for the BatchNorm that follows (statistics pass
// fused into the convolution); the stride-2 dgrad parity classes, whose output pixels are strided, stage the tile the same way
// and then store each pixel row with 16-byte global stores.
//
// Reference counterpart: the strided nn.Conv2d layers of src/model_ops/resnet.py:14-64 (downsampling blocks + shortcuts).
#include <cstdio>
#include <cstdlib>

#include "conv_epilogue.cuh"
#include "wgmma_common.cuh"

namespace {

using namespace tc;

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;
constexpr int NUM_THREADS = 256;
constexpr int MAX_TAPS = 9;
constexpr int MAX_CLASSES = 4;

struct TapConvArgs {
  int N, OH, OW;               // iteration space: one GEMM row per (n, i, j), tiled in BW x BH x BN patches
  int Cred, Cn;                // reduction channels per tap / output channels
  int BW, BH, BN;
  int in_mul;                  // input coordinate = patch origin * in_mul + tap offset   (stride for fprop, 1 for dgrad)
  int ntaps;                   // taps of ALL classes
  int tap_dw[MAX_TAPS], tap_dh[MAX_TAPS];
  int tap_wcol[MAX_TAPS];      // column of the tap inside a weight row (tap index * Cin)
  int out_H, out_W;            // output tensor geometry
  int out_mul;                 // output pixel = (i * out_mul + out_oh, j * out_mul + out_ow)
  // Output classes: ONE launch covers every parity class of a strided dgrad.  Class c owns taps [cls_tap0[c], cls_tap0[c+1]) and
  // writes the pixels (out_mul * i + cls_oh[c], out_mul * j + cls_ow[c]); tiles are numbered class-major, classes sorted by
  // decreasing tap count (longest tiles first: the static round-robin over CTAs then balances).  Dense launches have one class.
  int nclass;
  int cls_tap0[MAX_CLASSES + 1], cls_oh[MAX_CLASSES], cls_ow[MAX_CLASSES];
  // Thread-block cluster of cm x cn CTAs working on cm x cn neighbouring tiles (1 x 1 = no cluster).  The cn CTAs of a cluster
  // row share their activation tile and the cm CTAs of a column their weight tile: every CTA loads 1/cn of A and 1/cm of B and
  // TMA-multicasts it to the CTAs that need it, so the L2 -> SM traffic of a tile drops from A + B to A/cn + B/cm (these layers
  // are bound by exactly that traffic).  The cluster grid may overhang the layer (M or N tiles not a multiple of cm / cn): a CTA
  // whose tile lies beyond it still loads and multicasts its operand slices for its peers but stores nothing.
  int cm, cn;
  long long* dbg;              // optional per-CTA timeline (8 x int64, tools/prof_conv_timeline.py): null in production
  int sl_fw, sl_fh;            // the A slice of CTA column rn: split factors of the patch along w and h (n takes the rest)
  __nv_bfloat16* out;          // [N, out_H, out_W, Cn]
  const __nv_bfloat16* resid;  // optional tensor of the output's shape added in the epilogue (dgrad: the gradient of the other
                               // branch of a fork -- the residual shortcut -- so that autograd's separate add kernel disappears)
  const float* bias_f32;
  const __nv_bfloat16* bias_bf16;
  convepi::BnStatArgs stat;    // BatchNorm statistics of the output (TMA-store epilogue only)
};

// MODE 0: one CTA per tile.  MODE 1: multicast cluster (see TapConvArgs::cm).
// tmap_xs / tmap_ws: the same tensors with the SLICE boxes (1/cn of the patch, 1/cm of the weight rows).
constexpr int MODE_PLAIN = 0, MODE_MCAST = 1;

// Releases a consumed stage: every warp of the MMA warpgroup arrives once on the stage's empty barrier of every CTA that filled
// it (cluster: the CTAs of my row and column multicast into it; mask bit i = cluster rank i).
__device__ __forceinline__ void release_stage(uint64_t* bar, bool cluster, uint32_t mask, int lane) {
  if (lane != 0) return;
  if (!cluster) { mbar_arrive(bar); return; }
  for (uint32_t m = mask; m; m &= m - 1) mbar_arrive_cluster(bar, (uint32_t)__ffs(m) - 1u);
}

template <int BLOCK_N, int STAGES, bool B_MN, bool TMA_EPI, int MODE>
__global__ void __launch_bounds__(NUM_THREADS, 1)
convg_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                   const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_xs,
                   const __grid_constant__ CUtensorMap tmap_ws, const TapConvArgs a) {
  constexpr bool CLUSTER = MODE == MODE_MCAST;
  constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
  constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int EPI_BYTES = convepi::staging_bytes(BLOCK_N) + (TMA_EPI ? convepi::stat_bytes() : 0);

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sbuf = smem + STAGES * STAGE_BYTES;                                   // staging tile (1024-aligned: STAGE_BYTES % 1024 == 0)
  float* s_stat = reinterpret_cast<float*>(sbuf + convepi::staging_bytes(BLOCK_N));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + EPI_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  long long* dbg = a.dbg ? a.dbg + 8 * (long long)blockIdx.x : nullptr;
  if (dbg && threadIdx.x == 0) {
    unsigned long long gt;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
    dbg[0] = (long long)gt; dbg[1] = clock64();
  }
  const int wt = a.OW / a.BW, ht = a.OH / a.BH, nt = (a.N + a.BN - 1) / a.BN;
  const int m_tiles = wt * ht * nt;
  const int n_tiles = (a.Cn + BLOCK_N - 1) / BLOCK_N;
  const int c_blocks = a.Cred / BLOCK_K;           // 64-channel slices per tap
  const bool want_stats = TMA_EPI && a.stat.partial != nullptr;
  // Work units: a unit is one tile, or (cluster variant) a super-tile of cm x cn tiles handled by one cluster in lockstep.
  // Units are numbered class-major; unit -> (class, M super-tile, N super-tile); this CTA takes tile (rm, rn) of the unit.
  const int cs = CLUSTER ? a.cm * a.cn : 1;
  const int crank = CLUSTER ? (int)cluster_rank() : 0;
  const int rm = CLUSTER ? crank / a.cn : 0, rn = CLUSTER ? crank % a.cn : 0;
  const int sn_tiles = CLUSTER ? (n_tiles + a.cn - 1) / a.cn : n_tiles;
  const int class_units = (CLUSTER ? (m_tiles + a.cm - 1) / a.cm : m_tiles) * sn_tiles;
  const int num_units = class_units * a.nclass;
  const int unit0 = blockIdx.x / cs, unit_step = gridDim.x / cs;
  auto decode = [&](int unit, int& cls, int& mt, int& n0) {
    cls = unit / class_units;
    const int cu = unit - cls * class_units;
    const int smt = cu / sn_tiles, snt = cu - smt * sn_tiles;
    mt = CLUSTER ? smt * a.cm + rm : smt;
    n0 = (CLUSTER ? snt * a.cn + rn : snt) * BLOCK_N;
  };
  // multicast masks: the CTAs of my cluster row (they receive my A slice) and of my cluster column (my B slice)
  uint16_t mask_row = 1, mask_col = 1;
  if (CLUSTER) {
    mask_row = (uint16_t)(((1u << a.cn) - 1u) << (rm * a.cn));
    mask_col = 0;
    for (int j = 0; j < a.cm; ++j) mask_col |= (uint16_t)(1u << (j * a.cn + rn));
  }

  if (warp == 0 && lane == 0) {
    prefetch_tmap(CLUSTER ? &tmap_xs : &tmap_x);
    prefetch_tmap(CLUSTER ? &tmap_ws : &tmap_w);
    if (TMA_EPI) prefetch_tmap(&tmap_out);
  }
  if (warp == 1 && lane == 0) {
    // a slot is free again when every CTA that reads what I multicast into it has consumed it: my row and my column, 4 warps each
    const int releases = 4 * (CLUSTER ? a.cm + a.cn - 1 : 1);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], releases); }
    mbar_fence_init();
  }
  if (TMA_EPI && warp >= 4) {
    for (int i = threadIdx.x - 128; i < 2 * convepi::STAT_PARTS * convepi::STAT_MAX_C; i += convepi::EPI_THREADS) s_stat[i] = 0.f;
  }
  __syncthreads();
  if (CLUSTER) cluster_sync_all();                 // every barrier of the cluster is initialised before anyone signals a peer
  if (dbg && threadIdx.x == 0) dbg[2] = clock64();

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      int stage = 0; uint32_t phase = 0;
      // cluster variant: my slice of the activation patch (rows [rn * 128/cn, ...) of the tile) and of the weight tile
      const int a_rows = BLOCK_M / (CLUSTER ? a.cn : 1);
      const int sl_iw = rn % a.sl_fw, sl_ih = (rn / a.sl_fw) % a.sl_fh, sl_in = rn / (a.sl_fw * a.sl_fh);
      const int sl_fn = (CLUSTER ? a.cn : 1) / (a.sl_fw * a.sl_fh);
      const int sl_w = sl_iw * (a.BW / a.sl_fw), sl_h = sl_ih * (a.BH / a.sl_fh), sl_n = sl_in * (a.BN / sl_fn);
      const int b_rows = (B_MN ? BLOCK_K : BLOCK_N) / (CLUSTER ? a.cm : 1);
      for (int unit = unit0; unit < num_units; unit += unit_step) {
        int cls, mt, n0;
        decode(unit, cls, mt, n0);
        const int w0 = (mt % wt) * a.BW, h0 = ((mt / wt) % ht) * a.BH, nb0 = (mt / (wt * ht)) * a.BN;
        const int tap0 = a.cls_tap0[cls], k_blocks = (a.cls_tap0[cls + 1] - tap0) * c_blocks;
        for (int kb = 0; kb < k_blocks; ++kb) {
          const int tl = kb / c_blocks, c0 = (kb - tl * c_blocks) * BLOCK_K, tap = tap0 + tl;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + A_BYTES;
          mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
          if (!CLUSTER) {
            // activation patch of this tap: (strided) 4-D box, out-of-range pixels zero-filled by TMA
            tma_load_4d(sa, &tmap_x, c0, w0 * a.in_mul + a.tap_dw[tap], h0 * a.in_mul + a.tap_dh[tap], nb0, &full_bar[stage]);
            if (!B_MN) {
              tma_load_2d(sb, &tmap_w, a.tap_wcol[tap] + c0, n0, &full_bar[stage]);               // rows = Cout tile, K-major
            } else {
#pragma unroll
              for (int j = 0; j < BLOCK_N / 64; ++j)                                             // rows = Cout (K), cols = Cin (N)
                tma_load_2d(sb + j * (BLOCK_K * 128), &tmap_w, a.tap_wcol[tap] + n0 + 64 * j, c0, &full_bar[stage]);
            }
          } else {
            // the full barrier of EVERY destination CTA (same offset) receives the bytes; each CTA armed its own for A + B
            tma_load_4d_mc(sa + rn * a_rows * 128, &tmap_xs, c0, (w0 + sl_w) * a.in_mul + a.tap_dw[tap],
                           (h0 + sl_h) * a.in_mul + a.tap_dh[tap], nb0 + sl_n, &full_bar[stage], mask_row);
            if (!B_MN) {
              tma_load_2d_mc(sb + rm * b_rows * 128, &tmap_ws, a.tap_wcol[tap] + c0, n0 + rm * b_rows, &full_bar[stage], mask_col);
            } else {
#pragma unroll
              for (int j = 0; j < BLOCK_N / 64; ++j)
                tma_load_2d_mc(sb + j * (BLOCK_K * 128) + rm * b_rows * 128, &tmap_ws, a.tap_wcol[tap] + n0 + 64 * j,
                               c0 + rm * b_rows, &full_bar[stage], mask_col);
            }
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================== MMA + epilogue (one warpgroup) =====================
    const int et = threadIdx.x - 128;
    const uint32_t rel_mask = CLUSTER ? (uint32_t)(mask_row | mask_col) : 1u;
    int stage = 0; uint32_t phase = 0;
    float acc[2][BLOCK_N / 2];
    convepi::StatAcc<BLOCK_N> sacc;
    sacc.clear();
    // every tile of this CTA covers the same channels (one N tile, or one tile per CTA): statistics stay in registers until the end
    const bool stat_keep = sn_tiles == 1 || num_units <= unit_step;
    int stat_col0 = 0;
    for (int unit = unit0; unit < num_units; unit += unit_step) {
      int cls, mt, n0;
      decode(unit, cls, mt, n0);
      const int w0 = (mt % wt) * a.BW, h0 = ((mt / wt) % ht) * a.BH, nb0 = (mt / (wt * ht)) * a.BN;
      if (TMA_EPI && a.stat.bwd_x) {
        // BatchNorm-backward mode: pull this tile's rows of y (mask) and x into L2 before the MMAs of the tile --
        // they were written by the forward pass long ago and would otherwise cost a DRAM round trip per epilogue step
        const int rw = w0 + et % a.BW, rh = h0 + (et / a.BW) % a.BH, rn_ = nb0 + et / (a.BW * a.BH);
        if (rn_ < a.N) {
          const long long off = (((long long)rn_ * a.out_H + rh) * a.out_W + rw) * a.Cn + n0;
#pragma unroll
          for (int cb = 0; cb < BLOCK_N; cb += 64) {
            if (n0 + cb < a.Cn) {
              asm volatile("prefetch.global.L2 [%0];" ::"l"(a.stat.bwd_x + off + cb));
              if (a.stat.bwd_mask) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.stat.bwd_mask + off + cb));
            }
          }
        }
      }
      const int k_blocks = (a.cls_tap0[cls + 1] - a.cls_tap0[cls]) * c_blocks;
      if (dbg && et == 0 && unit == unit0) {                       // profiling: when did the first operands land?
        mbar_wait(&full_bar[stage], phase);
        dbg[3] = clock64();
      }
      int prev = -1;
      acc_undef<BLOCK_N / 2>(acc[0]);                             // the previous tile's values: dead during its epilogue
      acc_undef<BLOCK_N / 2>(acc[1]);
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
        mma_kblock<BLOCK_N, false, B_MN>(acc, sa, sa + A_BYTES, kb == 0);
        wgmma_wait<1>();                                           // the previous K block's MMAs have read their stage
        if (prev >= 0) release_stage(&empty_bar[prev], CLUSTER, rel_mask, lane);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      if (dbg && et == 0) dbg[4] = clock64();                      // last K block's wgmma issued
      wgmma_wait<0>();
      fence_acc<BLOCK_N / 2>(acc[0]);
      fence_acc<BLOCK_N / 2>(acc[1]);
      if (dbg && et == 0) dbg[5] = clock64();                      // accumulator complete
      release_stage(&empty_bar[prev], CLUSTER, rel_mask, lane);
      const bool tile_ok = mt < m_tiles && n0 < a.Cn;              // false: overhang of the cluster grid, nothing to store
      int valid_rows = tile_ok ? (a.N - nb0) * a.BW * a.BH : 0;    // rows are pixels, w fastest: the real ones are a prefix
      if (valid_rows > BLOCK_M) valid_rows = BLOCK_M;
      if (TMA_EPI) {
        // element offset of channel 0 of tile row r in a tensor of the output's shape
        auto row_off = [&](int r) -> long long {
          const int rw = w0 + r % a.BW, rh = h0 + (r / a.BW) % a.BH, rn_ = nb0 + r / (a.BW * a.BH);
          return (((long long)rn_ * a.out_H + rh) * a.out_W + rw) * a.Cn;
        };
        convepi::drain_tile<BLOCK_N>(acc, sbuf, et, valid_rows, n0, a.Cn, a.bias_f32, a.bias_bf16, a.resid, a.stat.bwd_mask, row_off);
        if (et == 0 && tile_ok) {
#pragma unroll
          for (int j = 0; j < BLOCK_N / 64; ++j)
            if (n0 + 64 * j < a.Cn) tma_store_4d(&tmap_out, sbuf + j * (128 * 128), n0 + 64 * j, w0, h0, nb0);
          tma_store_commit();
        }
        if (want_stats && tile_ok) {
          if (a.stat.bwd_x) sacc.add_tile_bwd(sbuf, et, valid_rows, a.stat.bwd_x, row_off, n0, a.Cn, a.stat.bwd_mean, a.stat.bwd_invstd);
          else sacc.add_tile(sbuf, et, valid_rows);
          stat_col0 = n0;
          if (!stat_keep) sacc.flush(s_stat, et, n0, a.Cn);
        }
      } else {
        // strided output pixels (stride-2 dgrad parity class): the same staged tile, then every thread stores its row (pixel
        // (out_mul * i + cls_oh, out_mul * j + cls_ow)) with 16-byte global stores
        auto row_off = [&](int r) -> long long {
          const int pw = w0 + r % a.BW, ph = h0 + (r / a.BW) % a.BH, pn = nb0 + r / (a.BW * a.BH);
          return (((long long)pn * a.out_H + (ph * a.out_mul + a.cls_oh[cls])) * a.out_W + (pw * a.out_mul + a.cls_ow[cls])) * a.Cn;
        };
        convepi::drain_tile<BLOCK_N>(acc, sbuf, et, valid_rows, n0, a.Cn, a.bias_f32, a.bias_bf16, a.resid, nullptr, row_off);
        if (et < valid_rows) {
          __nv_bfloat16* orow = a.out + row_off(et) + n0;
#pragma unroll
          for (int j = 0; j < BLOCK_N / 64; ++j) {
            if (n0 + 64 * j < a.Cn) {
#pragma unroll
              for (int c = 0; c < 8; ++c)
                *reinterpret_cast<uint4*>(orow + 64 * j + 8 * c) =
                    *reinterpret_cast<const uint4*>(sbuf + j * (128 * 128) + et * 128 + ((c ^ (et & 7)) << 4));
            }
          }
        }
      }
    }
    if (want_stats && stat_keep) sacc.flush(s_stat, et, stat_col0, a.Cn);
    if (TMA_EPI && et == 0) tma_store_wait<0>();                 // every tile of this CTA is in global memory
    if (dbg && et == 0) dbg[6] = clock64();                        // every tile of this CTA stored
  }

  __syncthreads();
  if (CLUSTER) cluster_sync_all();                 // no CTA leaves while a peer may still write into it or signal its barriers
  if (dbg && threadIdx.x == 0) {
    unsigned long long gt;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
    dbg[7] = (long long)gt;                                        // exit (before the statistics ticket / fold, if any)
  }
  if (want_stats) {
    // one tile per CTA (units <= clusters): slot = M tile, this CTA owns its N-tile's channels; otherwise slot = CTA, all channels
    const bool one_tile = num_units <= unit_step;
    int cls0, mt, n0;
    decode(unit0, cls0, mt, n0);
    if (one_tile && !(mt < m_tiles && n0 < a.Cn)) return;         // an overhanging CTA owns no slot and takes no ticket
    const int c_hi = n0 + BLOCK_N < a.Cn ? n0 + BLOCK_N : a.Cn;
    // one tile per CTA: the CTAs of one channel tile share a ticket and its last CTA folds only that tile's channels (the n_tiles
    // folds run in parallel); otherwise one ticket for the grid and the last CTA folds every channel
    convepi::finalize_stats<NUM_THREADS>(a.stat, s_stat, convepi::STAT_PARTS, a.Cn, one_tile ? mt : (int)blockIdx.x,
                                         one_tile ? m_tiles : (int)gridDim.x, one_tile ? n0 : 0, one_tile ? c_hi : a.Cn,
                                         reinterpret_cast<float*>(sbuf), one_tile ? n0 / BLOCK_N : 0, one_tile ? m_tiles : -1);
  }
}



struct WgradGArgs {
  int N, H, W, Cin, Cout;      // H, W: spatial size of dy (the K-block patch lives in dy space)
  int ks, stride, pad;         // filter size (1 or 3), stride, padding of the forward convolution
  int PW, PH, PN;               // 64-pixel patch shape
  int splits;                   // K splits
  float* partial;               // [splits][Cout][9*Cin]
};

template <int BLOCK_N, int STAGES>
__global__ void __launch_bounds__(NUM_THREADS, 1)
convg_wgrad_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_dy, const __grid_constant__ CUtensorMap tmap_x, const WgradGArgs a) {
  constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;            // 2 atoms of [64 px][64 co]
  constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wt = a.W / a.PW, ht = a.H / a.PH, nt = (a.N + a.PN - 1) / a.PN;
  const int k_total = wt * ht * nt;                          // 64-pixel K-blocks
  const int m_tiles = (a.Cout + BLOCK_M - 1) / BLOCK_M, n_tiles = (a.Cin + BLOCK_N - 1) / BLOCK_N;
  const int ntaps = a.ks * a.ks;
  const int out_tiles = m_tiles * ntaps * n_tiles;
  const int num_work = out_tiles * a.splits;
  const int k_per_split = (k_total + a.splits - 1) / a.splits;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmap_dy);
    prefetch_tmap(&tmap_x);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }
    mbar_fence_init();
  }
  __syncthreads();

  // work item -> (split, m tile, tap, n tile); splits of one output tile are spread over different CTAs
  auto decode = [&](int wi, int& split, int& co0, int& tap, int& ci0) {
    split = wi / out_tiles;
    int t = wi - split * out_tiles;
    const int ntile = t % n_tiles; t /= n_tiles;
    tap = t % ntaps; t /= ntaps;
    co0 = t * BLOCK_M; ci0 = ntile * BLOCK_N;
  };

  if (warp == 0) {
    if (elect_one()) {
      int stage = 0; uint32_t phase = 0;
      for (int wi = blockIdx.x; wi < num_work; wi += gridDim.x) {
        int split, co0, tap, ci0; decode(wi, split, co0, tap, ci0);
        const int r = tap / a.ks, s = tap - a.ks * r;
        const int kb0 = split * k_per_split, kb1 = min(k_total, kb0 + k_per_split);
        for (int kb = kb0; kb < kb1; ++kb) {
          const int w0 = (kb % wt) * a.PW, h0 = ((kb / wt) % ht) * a.PH, n0 = (kb / (wt * ht)) * a.PN;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + A_BYTES;
          // a 64-channel atom entirely beyond Cout is never read back: skip its load (its accumulator rows hold junk)
          const int a_atoms = min(BLOCK_M / 64, (a.Cout - co0 + 63) / 64);
          mbar_expect_tx(&full_bar[stage], a_atoms * (BLOCK_K * 128) + B_BYTES);
          for (int j = 0; j < a_atoms; ++j) tma_load_4d(sa + j * (BLOCK_K * 128), &tmap_dy, co0 + 64 * j, w0, h0, n0, &full_bar[stage]);
#pragma unroll
          for (int j = 0; j < BLOCK_N / 64; ++j) tma_load_4d(sb + j * (BLOCK_K * 128), &tmap_x, ci0 + 64 * j, w0 * a.stride + s - a.pad, h0 * a.stride + r - a.pad, n0, &full_bar[stage]);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    const int et = threadIdx.x - 128;
    int stage = 0; uint32_t phase = 0;
    float acc[2][BLOCK_N / 2];
    const long long row_pitch = (long long)ntaps * a.Cin;
    for (int wi = blockIdx.x; wi < num_work; wi += gridDim.x) {
      int split, co0, tap, ci0; decode(wi, split, co0, tap, ci0);
      const int kb0 = split * k_per_split, kb1 = min(k_total, kb0 + k_per_split);
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
        mma_kblock<BLOCK_N, true, true>(acc, sa, sa + A_BYTES, kb == kb0);    // both operands MN-major
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      fence_acc<BLOCK_N / 2>(acc[0]);
      fence_acc<BLOCK_N / 2>(acc[1]);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      // fp32 partial straight from the fragment: float2 stores of rows co0 + frag_row, columns ci0 + frag_col; an empty K range
      // (more splits than K-blocks) must still produce zeros
      const bool empty = kb1 <= kb0;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int co = co0 + frag_row(et, h, rr);
          if (co >= a.Cout) continue;
          float* orow = a.partial + ((long long)split * a.Cout + co) * row_pitch + (long long)tap * a.Cin;
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            const int ci = ci0 + frag_col(et, j);
            if (ci < a.Cin)
              *reinterpret_cast<float2*>(orow + ci) =
                  empty ? make_float2(0.f, 0.f) : make_float2(acc[h][4 * j + 2 * rr], acc[h][4 * j + 2 * rr + 1]);
          }
        }
      }
    }
  }
}

__global__ void wgradg_reduce_kernel(const float* partial, int splits, long long elems, __nv_bfloat16* out) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= elems) return;
  float4 acc = *reinterpret_cast<const float4*>(partial + i);
  for (int s = 1; s < splits; ++s) {                           // fixed order: bit-deterministic
    float4 v = *reinterpret_cast<const float4*>(partial + (long long)s * elems + i);
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  __nv_bfloat162 lo = __floats2bfloat162_rn(acc.x, acc.y), hi = __floats2bfloat162_rn(acc.z, acc.w);
  uint2 o;
  o.x = *reinterpret_cast<uint32_t*>(&lo); o.y = *reinterpret_cast<uint32_t*>(&hi);
  *reinterpret_cast<uint2*>(out + i) = o;
}

template <int BLOCK_N, bool B_MN, bool TMA_EPI, int MODE>
int launch_g(const CUtensorMap& tx, const CUtensorMap& tw, const CUtensorMap& tout, const CUtensorMap& txs, const CUtensorMap& tws,
             const TapConvArgs& a, int grid, cudaStream_t stream) {
  constexpr int STAGE_BYTES = BLOCK_M * BLOCK_K * 2 + BLOCK_N * BLOCK_K * 2;
  constexpr int EPI_BYTES = convepi::staging_bytes(BLOCK_N) + (TMA_EPI ? convepi::stat_bytes() : 0);
  constexpr int BUDGET = 220 * 1024 - EPI_BYTES;                         // 227 KB per block on H100, minus alignment + barriers
  constexpr int STAGES = BUDGET / STAGE_BYTES > 8 ? 8 : BUDGET / STAGE_BYTES;
  constexpr int SMEM = STAGES * STAGE_BYTES + EPI_BYTES + 1024 + 256;
  auto kern = convg_wgmma_kernel<BLOCK_N, STAGES, B_MN, TMA_EPI, MODE>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(NUM_THREADS); cfg.dynamicSmemBytes = SMEM; cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = MODE != MODE_PLAIN ? a.cm * a.cn : 1; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = MODE != MODE_PLAIN ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, tx, tw, tout, txs, tws, a);
  return e != cudaSuccess ? (int)e : (int)cudaGetLastError();
}

template <bool B_MN, bool TMA_EPI>
int launch_n(int block_n, int mode, const CUtensorMap& tx, const CUtensorMap& tw, const CUtensorMap& tout, const CUtensorMap& txs,
             const CUtensorMap& tws, const TapConvArgs& a, int grid, cudaStream_t stream) {
  if (mode == MODE_MCAST)
    return block_n == 64 ? launch_g<64, B_MN, TMA_EPI, MODE_MCAST>(tx, tw, tout, txs, tws, a, grid, stream)
                         : launch_g<128, B_MN, TMA_EPI, MODE_MCAST>(tx, tw, tout, txs, tws, a, grid, stream);
  return block_n == 64 ? launch_g<64, B_MN, TMA_EPI, MODE_PLAIN>(tx, tw, tout, txs, tws, a, grid, stream)
                       : launch_g<128, B_MN, TMA_EPI, MODE_PLAIN>(tx, tw, tout, txs, tws, a, grid, stream);
}

// patch shape for an iteration space of OH x OW pixels per image: BW * BH * BN == pixels with BW | OW and BH | OH (the largest
// power-of-two divisors that fit), so ANY image size tiles exactly -- 32 x 32 gives 32 x 4 x 1, 56 x 56 (ImageNet ResNets)
// 8 x 8 x 2, 14 x 14 gives 2 x 2 x 32 and 7 x 7 one pixel of 128 images.
int pow2_divisor(int v, int cap) {
  int d = 1;
  while (d * 2 <= cap && v % (d * 2) == 0) d *= 2;
  return d;
}
void patch_shape(int OH, int OW, int pixels, int& BW, int& BH, int& BN) {
  BW = pow2_divisor(OW, pixels);
  BH = pow2_divisor(OH, pixels / BW);
  BN = pixels / (BW * BH);
}

// Tile width, cluster shape and grid of one launch.
//
// The multicast cluster variant reproduces the plain kernel bit for bit; whether it is faster has not been measured on H100, so
// the default plan is cm = cn = 1 with the tile width chosen by the model below; DRACO_CONV_CLUSTER="cm,cn[,block_n]" forces a
// cluster shape ("auto" lets the model pick one) for experiments and for the tests that keep the multicast path honest.
// Model: a tile costs k_blocks * (A/cn + B/cm) bytes of L2 -> SM traffic and k_blocks * 4 MMAs of BLOCK_N/2 clocks.
struct TapPlan { int block_n, cm, cn, grid, units, mode; };

int clusters_resident(int cs, int num_sms) {
  // GPCs of an H100 expose 16-18 SMs each and a cluster never spans GPCs: count conservatively
  if (cs <= 1) return num_sms;
  if (cs == 2) return num_sms / 2 - 2;
  if (cs == 4) return num_sms / 4 - 3;
  return num_sms / 8 - 2;
}

TapPlan plan_tap(int m_tiles, int Cn, int k_blocks_total, int nclass, bool b_mn, int num_sms) {
  int f_cm = 1, f_cn = 1, f_bn = Cn >= 128 ? 128 : 64;          // default: no cluster, 128-wide tiles when the layer has them
  if (const char* e = getenv("DRACO_CONV_CLUSTER")) {
    int x = 0, y = 0, z = 0;
    const int got = sscanf(e, "%d,%d,%d", &x, &y, &z);
    if (got >= 2) { f_cm = x; f_cn = y; f_bn = -1; }
    else if (e[0] == 'a') { f_cm = f_cn = f_bn = -1; }
    if (got >= 3) f_bn = z;
  }
  TapPlan best = {Cn >= 128 ? 128 : 64, 1, 1, 0, 0, MODE_PLAIN};
  double best_t = 1e30;
  for (int bn = 128; bn >= 64; bn -= 64) {
    if (bn > Cn && bn != 64) continue;
    if (f_bn > 0 && bn != f_bn) continue;
    const int n_tiles = (Cn + bn - 1) / bn;
    for (int cm = 1; cm <= 8; cm *= 2) {
      for (int cn = 1; cm * cn <= 8; cn *= 2) {
        if (f_cm > 0 && (cm != f_cm || cn != f_cn)) continue;
        // a cluster may overhang the layer, but an operand it multicasts must be shared by at least two real tiles
        if ((cm > 1 && m_tiles < 2) || (cn > 1 && n_tiles < 2)) continue;
        if ((b_mn ? BLOCK_K : bn) / cm < 8 || BLOCK_M / cn < 8) continue;
        if (Cn % bn && cm * cn > 1) continue;                       // partial N tiles only without clusters
        const int cs = cm * cn;
        const long long units = (long long)((m_tiles + cm - 1) / cm) * ((n_tiles + cn - 1) / cn) * nclass;
        const long long clusters = units < clusters_resident(cs, num_sms) ? units : clusters_resident(cs, num_sms);
        const double waves = (double)((units + clusters - 1) / clusters);
        const double kb = (double)k_blocks_total / nclass;          // mean K blocks of a tile
        const double tile_bytes = kb * (16384.0 / cn + bn * 128.0 / cm);
        const double t_mma = waves * kb * 4 * (bn / 2);
        const double t_sm = waves * tile_bytes / 64.0;
        const double t_chip = (double)units * cs * tile_bytes / 6300.0;
        double t = t_mma > t_sm ? t_mma : t_sm;
        if (t_chip > t) t = t_chip;
        t += waves * 600 + (cs > 1 ? 400 : 0);                      // epilogue tail per wave, cluster launch + syncs
        if (t < best_t) { best_t = t; best = {bn, cm, cn, (int)(clusters * cs), (int)units, cs > 1 ? MODE_MCAST : MODE_PLAIN}; }
      }
    }
  }
  return best;
}

// slice boxes of the cluster variant: the patch BW x BH x BN split cn ways along n, then h, then w (rows of a slice stay contiguous)
void slice_shape(int BW, int BH, int BN, int cn, int& fw, int& fh, int& fn) {
  fn = cn < BN ? cn : BN;
  fh = cn / fn < BH ? cn / fn : BH;
  fw = cn / (fn * fh);
}

}  // namespace

// The tap table of one launch (also exported so that the host-side algebra can be tested without a GPU).
//   fprop            : every filter tap (r, s); input pixel = output pixel * stride + (r - pad, s - pad)
//   dgrad, class (ph, pw): output pixel (stride*i + ph, stride*j + pw) receives dy[i + dh, j + dw] * W[r, s] from the taps with
//                      (ph + pad - r) and (pw + pad - s) divisible by the stride; dh = (ph + pad - r) / stride, dw likewise
// Returns the number of taps; tap_index[t] = r * ks + s.
extern "C" int drc_convg_taps(int ks, int stride, int dgrad, int ph, int pw, int* dh, int* dw, int* tap_index) {
  const int pad = ks / 2;
  int n = 0;
  for (int rr = 0; rr < ks; ++rr) {
    for (int ss = 0; ss < ks; ++ss) {
      if (!dgrad) {
        dh[n] = rr - pad; dw[n] = ss - pad;
      } else {
        if ((ph + pad - rr) % stride || (pw + pad - ss) % stride) continue;
        dh[n] = (ph + pad - rr) / stride; dw[n] = (pw + pad - ss) / stride;
      }
      tap_index[n++] = rr * ks + ss;
    }
  }
  return n;
}

// 1 if the forward geometry x[N,H,W,Cin] -> y[N,H/stride,W/stride,Cout] (ks x ks filter, pad ks/2) is served.
extern "C" int drc_convg_supported(int H, int W, int Cin, int Cout, int ks, int stride) {
  if (!(ks == 1 || ks == 3) || !(stride == 1 || stride == 2)) return 0;
  if (H % stride || W % stride) return 0;
  const int OH = H / stride, OW = W / stride;
  if (OW < 1 || OH < 1 || OW > 4096 || OH > 4096) return 0;
  if (Cin % 64 || Cout % 64) return 0;
  return 1;
}

// fprop (dgrad == 0): act = x [N,H,W,Cin]      -> out = y  [N,H/stride,W/stride,Cout]
// dgrad (dgrad == 1): act = dy[N,H/s,W/s,Cout] -> out = dx [N,H,W,Cin]
// wgt: [Cout, ks, ks, Cin] bf16 (arena layout).  H, W are always the spatial size of the forward INPUT x.
// tma_store: 1 = staged TMA-store epilogue where the output is dense (everything but the stride-2 dgrad parity classes).
// stat_*: optional BatchNorm statistics of y (fprop + TMA-store epilogue only): workspace of drc_convg_stat_slots() * 2 * Cout
// floats, a zeroed ticket counter, outputs mean / invstd [Cout], optional running statistics (momentum update).
extern "C" int drc_convg_stat_slots(int N, int H, int W, int Cout, int stride, int num_sms) {
  // the number of partial-statistics slots only has to be an upper bound of what the launch uses (one slot per M tile when every
  // tile has its own CTA, one per CTA otherwise); the kernel is told the exact number
  const int OH = H / stride, OW = W / stride;
  int BW, BH, BN;
  patch_shape(OH, OW, BLOCK_M, BW, BH, BN);
  const int m_tiles = (OW / BW) * (OH / BH) * ((N + BN - 1) / BN);
  return m_tiles > num_sms ? m_tiles : num_sms;
}

// Test hook: the plan (block_n, cm, cn, grid, mode: 0 plain / 1 multicast cluster) the launcher would use (5 ints).
extern "C" int drc_convg_plan(int N, int H, int W, int Cin, int Cout, int ks, int stride, int dgrad, int num_sms, int* out4) {
  if (!drc_convg_supported(H, W, Cin, Cout, ks, stride)) return -1;
  const int OH = H / stride, OW = W / stride;
  int BW, BH, BN;
  patch_shape(OH, OW, BLOCK_M, BW, BH, BN);
  const int m_tiles = (OW / BW) * (OH / BH) * ((N + BN - 1) / BN);
  const int Cred = dgrad ? Cout : Cin, Cn = dgrad ? Cin : Cout;
  const bool strided_dgrad = dgrad && stride > 1;
  int nclass = 1, ntaps = ks * ks;
  if (strided_dgrad) { nclass = ks == 1 ? 1 : stride * stride; ntaps = ks * ks; }
  const TapPlan p = plan_tap(m_tiles, Cn, ntaps * (Cred / BLOCK_K), nclass, dgrad != 0, num_sms);
  out4[0] = p.block_n; out4[1] = p.cm; out4[2] = p.cn; out4[3] = p.grid; out4[4] = p.mode;
  return 0;
}

static inline bool dense_out_of(int dgrad, int stride) { return !(dgrad && stride > 1); }

// Test / profiling hook: the next drc_convg launches write their per-CTA timeline (8 x int64 per CTA) here; null disables.
static long long* g_convg_dbg = nullptr;
extern "C" void drc_convg_set_timeline(long long* buf) { g_convg_dbg = buf; }


extern "C" int drc_convg(const void* act, const void* wgt, void* out, int N, int H, int W, int Cin, int Cout, int ks, int stride,
                         int dgrad, const float* bias_f32, const void* bias_bf16, const void* resid, int tma_store, float* stat_partial,
                         unsigned int* stat_counter, float* stat_mean, float* stat_invstd, float* running_mean, float* running_var,
                         float eps, float momentum, const void* bwd_x, const void* bwd_mask, const float* bwd_mean,
                         const float* bwd_invstd, float* bwd_sums, float* bwd_dgamma, float* bwd_dbeta, int num_sms, int device,
                         cudaStream_t stream) {
  if (!drc_convg_supported(H, W, Cin, Cout, ks, stride)) return -1;
  if (device >= 0) { cudaError_t e = cudaSetDevice(device); if (e != cudaSuccess) return (int)e; }
  const int OH = H / stride, OW = W / stride;
  TapConvArgs a;
  a.N = N; a.OH = OH; a.OW = OW;                 // both passes iterate over an OH x OW grid per image (dgrad: per parity class)
  a.Cred = dgrad ? Cout : Cin; a.Cn = dgrad ? Cin : Cout;
  patch_shape(OH, OW, BLOCK_M, a.BW, a.BH, a.BN);
  a.out = (__nv_bfloat16*)out; a.bias_f32 = bias_f32; a.bias_bf16 = (const __nv_bfloat16*)bias_bf16;
  a.resid = (const __nv_bfloat16*)resid;
  if (resid && !dense_out_of(dgrad, stride) && ks == 1) return -6;      // 1x1 / stride 2 dgrad leaves pixels to the memset
  a.stat.partial = nullptr; a.stat.counter = stat_counter; a.stat.mean = stat_mean; a.stat.invstd = stat_invstd;
  a.stat.running_mean = running_mean; a.stat.running_var = running_var; a.stat.count = (long long)N * OH * OW;
  a.stat.eps = eps; a.stat.momentum = momentum;
  a.stat.bwd_x = (const __nv_bfloat16*)bwd_x; a.stat.bwd_mask = (const __nv_bfloat16*)bwd_mask; a.stat.bwd_mean = bwd_mean;
  a.stat.bwd_invstd = bwd_invstd; a.stat.bwd_sums = bwd_sums; a.stat.bwd_dgamma = bwd_dgamma; a.stat.bwd_dbeta = bwd_dbeta;
  const bool dense_out = !(dgrad && stride > 1);
  const bool tma_epi = tma_store && dense_out;
  if (bwd_x && !(stat_partial && dgrad && bwd_mean && bwd_invstd && bwd_sums && bwd_dgamma && bwd_dbeta)) return -7;
  if (stat_partial) {
    // forward statistics of y (fprop) or BatchNorm-backward sums of the layer that fed this convolution (dgrad + bwd_x)
    if ((dgrad != 0) != (bwd_x != nullptr) || !tma_epi || a.Cn > convepi::STAT_MAX_C || (a.Cn & 3)) return -4;
    a.stat.partial = stat_partial;
  } else {
    a.stat.bwd_mask = nullptr;
  }
  const int m_tiles = (OW / a.BW) * (OH / a.BH) * ((N + a.BN - 1) / a.BN);

  // ---- tap table (+ output classes)
  a.in_mul = dgrad ? 1 : stride;
  a.out_H = dgrad ? H : OH; a.out_W = dgrad ? W : OW; a.out_mul = dgrad ? stride : 1;
  if (dgrad) { a.bias_f32 = nullptr; a.bias_bf16 = nullptr; }
  if (dense_out) {
    int tidx[MAX_TAPS];
    a.ntaps = drc_convg_taps(ks, dgrad ? 1 : stride, dgrad, 0, 0, a.tap_dh, a.tap_dw, tidx);
    for (int t = 0; t < a.ntaps; ++t) a.tap_wcol[t] = tidx[t] * Cin;
    a.nclass = 1; a.cls_tap0[0] = 0; a.cls_tap0[1] = a.ntaps; a.cls_oh[0] = a.cls_ow[0] = 0;
  } else {
    // stride 2 dgrad: the s x s parity classes of dx in ONE launch (class-major unit list, longest classes first)
    struct Cls { int ph, pw, n, dh[MAX_TAPS], dw[MAX_TAPS], tidx[MAX_TAPS]; } cls[MAX_CLASSES];
    int nc = 0, empty = 0;
    for (int ph = 0; ph < stride; ++ph)
      for (int pw = 0; pw < stride; ++pw) {
        Cls c; c.ph = ph; c.pw = pw;
        c.n = drc_convg_taps(ks, stride, 1, ph, pw, c.dh, c.dw, c.tidx);
        if (c.n == 0) { ++empty; continue; }
        int at = nc++;
        while (at > 0 && cls[at - 1].n < c.n) { cls[at] = cls[at - 1]; --at; }
        cls[at] = c;
      }
    if (empty) {                                  // classes that receive nothing (1x1 / stride 2) have to read as zero
      cudaError_t e = cudaMemsetAsync(out, 0, (size_t)N * H * W * Cin * 2, stream);
      if (e != cudaSuccess) return (int)e;
    }
    a.nclass = nc; a.ntaps = 0;
    for (int c = 0; c < nc; ++c) {
      a.cls_tap0[c] = a.ntaps; a.cls_oh[c] = cls[c].ph; a.cls_ow[c] = cls[c].pw;
      for (int t = 0; t < cls[c].n; ++t, ++a.ntaps) {
        a.tap_dh[a.ntaps] = cls[c].dh[t]; a.tap_dw[a.ntaps] = cls[c].dw[t]; a.tap_wcol[a.ntaps] = cls[c].tidx[t] * Cin;
      }
    }
    a.cls_tap0[nc] = a.ntaps;
  }

  // ---- plan + tensor maps
  const TapPlan plan = plan_tap(m_tiles, a.Cn, a.ntaps * (a.Cred / BLOCK_K), a.nclass, dgrad != 0, num_sms);
  const int block_n = plan.block_n;
  a.cm = plan.cm; a.cn = plan.cn; a.dbg = g_convg_dbg;
  int fw = 1, fh = 1, fn = 1;
  slice_shape(a.BW, a.BH, a.BN, a.cn, fw, fh, fn);
  a.sl_fw = fw; a.sl_fh = fh;
  CUtensorMap tx, tw, tout, txs, tws;
  const long long wcols = (long long)ks * ks * Cin;               // weights as a matrix [Cout rows][ks*ks*Cin cols]
  int r = encode_mat(&tw, wgt, Cout, wcols, wcols, dgrad ? BLOCK_K : block_n);
  if (r) return 2000 + r;
  // MODE_MCAST: 1/cm of the weight tile's rows
  r = encode_mat(&tws, wgt, Cout, wcols, wcols, (dgrad ? BLOCK_K : block_n) / a.cm);
  if (r) return 2100 + r;
  const int aC = dgrad ? Cout : Cin, aW = dgrad ? OW : W, aH = dgrad ? OH : H, aS = dgrad ? 1 : stride;
  r = encode_act(&tx, act, aC, aW, aH, N, a.BW, a.BH, a.BN, aS);
  if (r) return 1000 + r;
  r = encode_act(&txs, act, aC, aW, aH, N, a.BW / fw, a.BH / fh, a.BN / fn, aS);
  if (r) return 1100 + r;
  tout = tw;                                      // placeholder when the direct epilogue is used (never dereferenced)
  if (tma_epi) {
    r = encode_act(&tout, out, a.Cn, a.out_W, a.out_H, N, a.BW, a.BH, a.BN, 1);
    if (r) return 3000 + r;
  }
  if (!dgrad) return tma_epi ? launch_n<false, true>(block_n, plan.mode, tx, tw, tout, txs, tws, a, plan.grid, stream)
                             : launch_n<false, false>(block_n, plan.mode, tx, tw, tout, txs, tws, a, plan.grid, stream);
  return tma_epi ? launch_n<true, true>(block_n, plan.mode, tx, tw, tout, txs, tws, a, plan.grid, stream)
                 : launch_n<true, false>(block_n, plan.mode, tx, tw, tout, txs, tws, a, plan.grid, stream);
}

namespace {
void wgrad_patch(int H, int W, int& PW, int& PH, int& PN) { patch_shape(H, W, 64, PW, PH, PN); }
}

// K splits and fp32 workspace elements.  H, W: spatial size of the forward input x.
extern "C" int drc_convg_wgrad_plan(int N, int H, int W, int Cin, int Cout, int ks, int stride, int num_sms, long long* ws_elems) {
  const int OH = H / stride, OW = W / stride, ntaps = ks * ks;
  const int block_n = Cin >= 128 ? 128 : 64;
  const int out_tiles = ((Cout + BLOCK_M - 1) / BLOCK_M) * ntaps * ((Cin + block_n - 1) / block_n);
  int PW, PH, PN;
  wgrad_patch(OH, OW, PW, PH, PN);
  const int k_total = (OW / PW) * (OH / PH) * ((N + PN - 1) / PN);
  int splits = num_sms / out_tiles;
  if (splits > k_total) splits = k_total;
  if (splits < 1) splits = 1;
  if (splits > 64) splits = 64;
  if (ws_elems) *ws_elems = (long long)splits * Cout * ntaps * Cin;
  return splits;
}

extern "C" int drc_convg_wgrad_supported(int H, int W, int Cin, int Cout, int ks, int stride) {
  if (!(ks == 1 || ks == 3) || !(stride == 1 || stride == 2)) return 0;
  if (H % stride || W % stride) return 0;
  const int OH = H / stride, OW = W / stride;
  if (OW < 1 || OH < 1 || OW > 4096 || OH > 4096) return 0;
  if (Cin % 64 || Cout % 64) return 0;
  return 1;
}

// dy: [N,H/s,W/s,Cout] bf16, x: [N,H,W,Cin] bf16 -> dw: [Cout,ks,ks,Cin] bf16 (arena layout).
extern "C" int drc_convg_wgrad(const void* dy, const void* x, void* dw, float* ws, int N, int H, int W, int Cin, int Cout, int ks,
                               int stride, int num_sms, int device, cudaStream_t stream) {
  if (!drc_convg_wgrad_supported(H, W, Cin, Cout, ks, stride)) return -1;
  if (device >= 0) { cudaError_t e = cudaSetDevice(device); if (e != cudaSuccess) return (int)e; }
  const int OH = H / stride, OW = W / stride, ntaps = ks * ks;
  WgradGArgs a;
  a.N = N; a.H = OH; a.W = OW; a.Cin = Cin; a.Cout = Cout; a.ks = ks; a.stride = stride; a.pad = ks / 2;
  wgrad_patch(OH, OW, a.PW, a.PH, a.PN);
  a.splits = drc_convg_wgrad_plan(N, H, W, Cin, Cout, ks, stride, num_sms, nullptr);
  a.partial = ws;
  const int block_n = Cin >= 128 ? 128 : 64;
  CUtensorMap tdy, tx;
  int r = encode_act(&tdy, dy, Cout, OW, OH, N, a.PW, a.PH, a.PN, 1);
  if (r) return 1000 + r;
  r = encode_act(&tx, x, Cin, W, H, N, a.PW, a.PH, a.PN, stride);
  if (r) return 2000 + r;
  const int out_tiles = ((Cout + BLOCK_M - 1) / BLOCK_M) * ntaps * ((Cin + block_n - 1) / block_n);
  const int work = out_tiles * a.splits;
  const int grid = work < num_sms ? work : num_sms;
  if (block_n == 64) {
    constexpr int BN_ = 64, SB = BLOCK_M * BLOCK_K * 2 + BN_ * BLOCK_K * 2, ST = (200 * 1024) / SB > 8 ? 8 : (200 * 1024) / SB;
    constexpr int SM = ST * SB + 1280;
    auto kern = convg_wgrad_wgmma_kernel<BN_, ST>;
    static bool cfgd = false;
    if (!cfgd) { cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SM); if (e != cudaSuccess) return (int)e; cfgd = true; }
    kern<<<grid, NUM_THREADS, SM, stream>>>(tdy, tx, a);
  } else {
    constexpr int BN_ = 128, SB = BLOCK_M * BLOCK_K * 2 + BN_ * BLOCK_K * 2, ST = (200 * 1024) / SB > 8 ? 8 : (200 * 1024) / SB;
    constexpr int SM = ST * SB + 1280;
    auto kern = convg_wgrad_wgmma_kernel<BN_, ST>;
    static bool cfgd = false;
    if (!cfgd) { cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SM); if (e != cudaSuccess) return (int)e; cfgd = true; }
    kern<<<grid, NUM_THREADS, SM, stream>>>(tdy, tx, a);
  }
  int rc = (int)cudaGetLastError();
  if (rc) return rc;
  const long long elems = (long long)Cout * ntaps * Cin;
  wgradg_reduce_kernel<<<(unsigned)((elems / 4 + 255) / 256), 256, 0, stream>>>(ws, a.splits, elems, (__nv_bfloat16*)dw);
  return (int)cudaGetLastError();
}
