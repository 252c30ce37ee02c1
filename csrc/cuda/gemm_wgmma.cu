// K10 (dense part): bf16 GEMM on the Hopper tensor cores, written directly against the sm_90a programming model -- TMA
// (cp.async.bulk.tensor) stages 128B-swizzled operand tiles in shared memory, one warpgroup issues wgmma with the fp32
// accumulator in registers and, once a tile is complete, applies bias / ReLU / down-conversion on the way to global memory,
// straight from the accumulator fragments (every thread stores its own column pairs).
//
//   C[M,N] = op(A) * op(B)^T   with  A: M x K,  B: N x K  (both described K-major *or* MN-major, so the
//   three products of a linear layer -- y = x W^T, dx = dy W, dW = dy^T x -- run without a transpose pass)
//
// Role layout (256 threads, one persistent CTA per SM, tiles strided over the grid):
//   warp 0     TMA producer      (one elected lane)
//   warps 4-7  MMA + epilogue    (one warpgroup: wgmma 64 x BLOCK_N x 16 on both 64-row halves of the 128-row tile)
// Pipeline: smem full/empty ring of STAGES stages; the producer runs ahead into the next tile while the epilogue drains this one.
//
// The reference has no counterpart (its dense math is PyTorch-0.3 CPU THNN); this is the engine behind
// draco_b200.ops.linear and the pointwise convolutions.
#include "wgmma_common.cuh"

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;           // 64 bf16 = 128 bytes = one swizzle-128B atom row
constexpr int NUM_THREADS = 256;

struct GemmArgs {
  int M, N, K;
  void* C;
  long long ldc;                      // elements
  int c_fp32;                         // 1: C is fp32, 0: bf16
  const float* bias_f32;              // optional bias[N]
  const __nv_bfloat16* bias_bf16;     // optional bias[N]
  int relu;
  int accumulate;                     // C += result (fp32 or bf16 read-modify-write)
};

using namespace tc;

// Tile rasterisation: groups of GROUP_M row blocks x all column blocks, column-major inside a group (the tiles in flight cover a
// roughly square block of the output: fewer distinct operand panels per wave -> better L2 reuse on large problems).
constexpr int GROUP_M = 8;
__device__ __forceinline__ void tile_coords(int tile, int m_blocks, int n_blocks, int& mb, int& nb) {
  const int per_group = GROUP_M * n_blocks;
  const int g = tile / per_group, first = g * GROUP_M;
  const int gm = (m_blocks - first) < GROUP_M ? (m_blocks - first) : GROUP_M;
  const int r = tile - g * per_group;
  mb = first + r % gm;
  nb = r / gm;
}

template <int BLOCK_N, int STAGES, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const GemmArgs args) {
  constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
  constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static_assert(!B_MN || BLOCK_N % 64 == 0, "MN-major B needs 64-wide atoms");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m_blocks = (args.M + BLOCK_M - 1) / BLOCK_M;
  const int n_blocks = (args.N + BLOCK_N - 1) / BLOCK_N;
  const int num_tiles = m_blocks * n_blocks;
  const int k_blocks = (args.K + BLOCK_K - 1) / BLOCK_K;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int mb_, nb_;
        tile_coords(tile, m_blocks, n_blocks, mb_, nb_);
        const int m0 = mb_ * BLOCK_M, n0 = nb_ * BLOCK_N;
        for (int kb = 0; kb < k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + A_BYTES;
          mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
          const int k0 = kb * BLOCK_K;
          if (!A_MN) tma_load_2d(sa, &tmap_a, k0, m0, &full_bar[stage]);
          else {
#pragma unroll
            for (int j = 0; j < BLOCK_M / 64; ++j) tma_load_2d(sa + j * (BLOCK_K * 128), &tmap_a, m0 + 64 * j, k0, &full_bar[stage]);
          }
          if (!B_MN) tma_load_2d(sb, &tmap_b, k0, n0, &full_bar[stage]);
          else {
#pragma unroll
            for (int j = 0; j < BLOCK_N / 64; ++j) tma_load_2d(sb + j * (BLOCK_K * 128), &tmap_b, n0 + 64 * j, k0, &full_bar[stage]);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================== MMA + epilogue (one warpgroup) =====================
    const int et = threadIdx.x - 128;                 // thread of the warpgroup: owns the fragment rows / columns of tc::frag_row / frag_col
    int stage = 0; uint32_t phase = 0;
    const bool vec_ok = (args.ldc % 8 == 0) && ((reinterpret_cast<uintptr_t>(args.C) & 15) == 0);
    float acc[2][BLOCK_N / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int mb_, nb_;
      tile_coords(tile, m_blocks, n_blocks, mb_, nb_);
      const int m0 = mb_ * BLOCK_M, n0 = nb_ * BLOCK_N;
      int prev = -1;
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
        mma_kblock<BLOCK_N, A_MN, B_MN>(acc, sa, sa + A_BYTES, kb == 0);
        wgmma_wait<1>();                                // the previous K block's MMAs have read their stage
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      fence_acc<BLOCK_N / 2>(acc[0]);
      fence_acc<BLOCK_N / 2>(acc[1]);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
      // epilogue straight from the fragment: column pairs (c, c + 1) of four rows per thread, 8- / 4-byte stores
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int row = m0 + frag_row(et, h, rr);
          if (row >= args.M) continue;
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            const int col = n0 + frag_col(et, j);
            if (col >= args.N) continue;
            float f[2] = {acc[h][4 * j + 2 * rr], acc[h][4 * j + 2 * rr + 1]};
            if (args.bias_f32 || args.bias_bf16) {
#pragma unroll
              for (int e = 0; e < 2; ++e)
                if (col + e < args.N) f[e] += args.bias_f32 ? args.bias_f32[col + e] : __bfloat162float(args.bias_bf16[col + e]);
            }
            if (args.relu) { f[0] = fmaxf(f[0], 0.f); f[1] = fmaxf(f[1], 0.f); }
            const bool pair = col + 1 < args.N && vec_ok && !args.accumulate;
            if (args.c_fp32) {
              float* dst = reinterpret_cast<float*>(args.C) + (long long)row * args.ldc + col;
              if (pair) {
                *reinterpret_cast<float2*>(dst) = make_float2(f[0], f[1]);
              } else {
#pragma unroll
                for (int e = 0; e < 2; ++e) if (col + e < args.N) dst[e] = args.accumulate ? dst[e] + f[e] : f[e];
              }
            } else {
              __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(args.C) + (long long)row * args.ldc + col;
              if (pair) {
                *reinterpret_cast<uint32_t*>(dst) = pack2(f[0], f[1]);
              } else {
#pragma unroll
                for (int e = 0; e < 2; ++e)
                  if (col + e < args.N) dst[e] = __float2bfloat16_rn(args.accumulate ? __bfloat162float(dst[e]) + f[e] : f[e]);
              }
            }
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// operand X: logical [rows(MN), K].  mn_major == 0: memory is [rows][ld] (K contiguous).  mn_major == 1: memory is [K][ld] (MN contiguous).
int make_tmap(CUtensorMap* out, const void* ptr, long long rows, long long K, long long ld, int mn_major, int box_rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return -1;
  cuuint64_t dims[2], strides[1];
  cuuint32_t box[2], estr[2] = {1, 1};
  if (!mn_major) { dims[0] = (cuuint64_t)K; dims[1] = (cuuint64_t)rows; box[0] = BLOCK_K; box[1] = (cuuint32_t)box_rows; }
  else           { dims[0] = (cuuint64_t)rows; dims[1] = (cuuint64_t)K; box[0] = 64; box[1] = BLOCK_K; }
  strides[0] = (cuuint64_t)ld * 2;
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return (int)r;
}

template <int BLOCK_N, bool A_MN, bool B_MN>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& g, int num_sms, cudaStream_t stream) {
  constexpr int STAGE_BYTES = BLOCK_M * BLOCK_K * 2 + BLOCK_N * BLOCK_K * 2;
  constexpr int BUDGET = 200 * 1024;
  constexpr int STAGES = BUDGET / STAGE_BYTES > 8 ? 8 : BUDGET / STAGE_BYTES;
  constexpr int SMEM = STAGES * STAGE_BYTES + 1024 + 256;
  auto kern = gemm_bf16_wgmma_kernel<BLOCK_N, STAGES, A_MN, B_MN>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  const int tiles = ((g.M + BLOCK_M - 1) / BLOCK_M) * ((g.N + BLOCK_N - 1) / BLOCK_N);
  const int grid = tiles < num_sms ? tiles : num_sms;
  kern<<<grid, NUM_THREADS, SMEM, stream>>>(ta, tb, g);
  return (int)cudaGetLastError();
}

template <int BLOCK_N>
int dispatch_major(int a_mn, int b_mn, const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& g, int sms, cudaStream_t s) {
  if (!a_mn && !b_mn) return launch<BLOCK_N, false, false>(ta, tb, g, sms, s);
  if (a_mn && !b_mn) return launch<BLOCK_N, true, false>(ta, tb, g, sms, s);
  if constexpr (BLOCK_N % 64 == 0) {
    if (!a_mn && b_mn) return launch<BLOCK_N, false, true>(ta, tb, g, sms, s);
    return launch<BLOCK_N, true, true>(ta, tb, g, sms, s);
  }
  return -2;
}

}  // namespace

// C[M,N] (+)= A * B^T.  a_mn / b_mn select the memory order of the operands (see make_tmap).
// Requirements: bf16 operands, 16-byte aligned bases, leading dimensions multiple of 8 elements.
extern "C" int drc_gemm_bf16(const void* A, long long lda, int a_mn, const void* B, long long ldb, int b_mn, void* C, long long ldc,
                             int c_fp32, int M, int N, int K, const float* bias_f32, const void* bias_bf16, int relu, int accumulate,
                             int block_n, int num_sms, int device, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  // autograd worker threads start without a bound context; the driver-API tensor-map encode needs one
  if (device >= 0) { cudaError_t e = cudaSetDevice(device); if (e != cudaSuccess) return (int)e; }
  if ((lda % 8) || (ldb % 8) || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15)) return -3;
  if (block_n == 0) {
    // 128 columns is the widest tile one warpgroup's registers hold (128 x 128 fp32 = 128 registers per thread)
    block_n = (N > 64) ? 128 : (N > 32 ? 64 : (b_mn ? 64 : 32));
  }
  if (block_n == 256) block_n = 128;                 // same products, register-sized tile (see above)
  if (b_mn && block_n < 64) block_n = 64;
  CUtensorMap ta, tb;
  int r = make_tmap(&ta, A, M, K, lda, a_mn, BLOCK_M);
  if (r) return 1000 + r;
  r = make_tmap(&tb, B, N, K, ldb, b_mn, block_n);
  if (r) return 2000 + r;
  GemmArgs g;
  g.M = M; g.N = N; g.K = K; g.C = C; g.ldc = ldc; g.c_fp32 = c_fp32; g.bias_f32 = bias_f32;
  g.bias_bf16 = reinterpret_cast<const __nv_bfloat16*>(bias_bf16); g.relu = relu; g.accumulate = accumulate;
  switch (block_n) {
    case 32: return dispatch_major<32>(a_mn, b_mn, ta, tb, g, num_sms, stream);
    case 64: return dispatch_major<64>(a_mn, b_mn, ta, tb, g, num_sms, stream);
    case 128: return dispatch_major<128>(a_mn, b_mn, ta, tb, g, num_sms, stream);
    default: return -4;
  }
}
