// K7 + K8 + K9 (+ the second half of K3 / K4 / K6): fused "aggregate -> optimizer (SGD-momentum | Adam | AMSGrad) -> parameter broadcast".
//
// Reference: the PS first builds the aggregated gradient per tensor (mean: baseline_master.py:267-269; vote
// winners summed per tensor: rep_master.py:154-168 -- here divided by #groups, a documented deviation, DESIGN.md section 7; Krum winner: baseline_master.py:278-296; Fourier recombination
// Re(v^T R)/n: cyclic_master.py:125-129,171-172), then SGDModified.step / AdamModified.step (optim/sgd_modified.py:53-88,
// optim/adam_modified.py:32-92), then
// one MPI.Bcast per tensor (baseline_master.py:180-186).  Here a single streaming kernel per step does all
// three: it reads only the gradient rows that contribute, updates momentum + fp32 master parameters in
// place, and stores the fresh parameters directly into every worker's parameter arena -- with one NVLS
// `multimem.st` through a multicast mapping when available, otherwise with unicast peer stores -- and the
// last CTA raises the step-stamped `params_ready` flag on every worker.  No NCCL call.
#include "common.cuh"

struct UpdateArgs {
  // gradient source ---------------------------------------------------------------------------
  int mode;                       // 0: select-sum over `select` table; 1: cyclic recombination; 2: real per-tensor weights;
                                  // 3: coordinate-wise trimmed mean over K rows (see `trim`);
                                  // 4: Bulyan's average of the K - 2 trim values nearest the coordinate median of K rows;
                                  // 5: centered clipping, v + sum_k w[tensor][k] (g_k - v) around the centre `center`;
                                  // 6: signSGD majority vote over the K = P sign rows (slots 0..K-1, K <= 32);
                                  // 7: mode 3 over the K = nb worker-bucket rows of `wb_mask` / `wb_scale`;
                                  // 8: mode 5 over those rows
  const float* grad_in;           // mode 0: [P][slot_stride] fp32 ; mode 1: [n][2*slot_stride] complex64 ;
                                  // mode 6: [K][slot_stride] uint32 sign words (bit b of word w = element 32w + b is < 0)
  long long slot_stride;          // elements (fp32 words for mode 0, complex elements for mode 1, uint32 sign words for mode 6)
  const int* select;              // modes 0, 2, 3: [K][T] worker slot to read for (k, tensor); null -> rows 0..K-1 for all
                                  // tensors.  DETOX: the vote's winner_slot table, so that the rule runs on the G group winners
  int K;                          // mode 0: rows summed per tensor ; mode 1: n workers
  float scale;                    // 1/K (mean, vote, multi-Krum), 1 (krum, median vector), 1/n (cyclic), 1/(K - 2 trim) (mode 3)
  const float2* recomb;           // mode 1: [T][n] recombination vector v (float2 = complex64); mode 2: float [T][K] weights
  TileView tv;
  // optimizer ---------------------------------------------------------------------------------
  float* params;                  // PS master fp32 [D]
  float* momentum;                // [D] SGD momentum buffer / Adam first moment
  float* exp_avg_sq;              // [D] Adam second moment (null for SGD)
  float* max_exp_avg_sq;          // [D] AMSGrad running maximum (null otherwise)
  const HyperParams* hp;
  const unsigned long long* step_ptr;
  unsigned long long first_step;  // step index at which momentum buffers are created (torch semantics)
  float* grad_out;                // optional: aggregated gradient written out (diagnostics / tests), may be null
  // broadcast ---------------------------------------------------------------------------------
  float* mc_params;               // NVLS multicast pointer to the params arena of every rank, or null
  float* dst[DRC_MAX_DST];        // unicast destinations (peer pointers to workers' params arenas)
  int ndst;
  unsigned int* done_counter;
  FlagList flags;                 // params_ready flags (peer pointers); value written = step + 1
  int tile_begin, tile_end;       // bucket of tiles to update + broadcast (tile_end == 0: whole arena)
  int trim;                       // mode 3: values dropped at each end of every coordinate (K = P <= TRIM_MAXP rows,
                                  // scale = 1 / (P - 2 * trim)); coordinate median: trim = (P - 1) / 2.  Mode 4: Bulyan's f
                                  // (K = theta = P - 2f selected rows, scale = 1 / (K - 2 * trim))
  // nearest-neighbour mixing in front of modes 3 and 4 (appended: the fields above keep their offsets) ------------------
  const unsigned int* mix;        // [mixP][T] neighbour masks of nnm_mix (bit j = raw row j is in N_i), or null: no mixing
  int mixP;                       // raw rows P (slots 0..P-1); mode 3 sorts K = P mixed rows, mode 4 the K = theta of `select`
  float mix_scale;                // fp32(1 / n_mix), n_mix = P - f
  // centered clipping (mode 5; appended) ------------------------------------------------------------------------------------
  float* center;                  // [D] the centre v, replaced by the aggregate g; weights in `recomb` as float [T][K]
  // worker buckets (mode 7; appended) ---------------------------------------------------------------------------------------
  const unsigned int* wb_mask;    // [K] member masks of the step's K = nb bucket rows (bit j = slot j), from wbucket_plan_kernel
  const float* wb_scale;          // [K] fp32(1 / |b|) of each bucket row
};

// ---------------------------------------------------------------------------------------------
// Mode 3: coordinate-wise trimmed mean (Yin et al., ICML 2018) and coordinate-wise median.
//
// Every thread sorts the P values of each of its 4 coordinates in registers with Batcher's odd-even merge network (N = 4,
// 8 or 16 inputs, padded with a sentinel), on order-preserving uint32 keys so that compare-exchange is an integer min/max:
// -Inf < finite < +Inf < NaN < padding.  NaN (any sign or payload) becomes the largest non-sentinel key, so up to `trim`
// NaN / +-Inf values per coordinate land in the trimmed tails.  The kept values are summed in ascending order in fp32:
// the result depends only on the P values of the coordinate, not on the grid or on the bucketing.
// ---------------------------------------------------------------------------------------------
#define TRIM_MAXP 16

__device__ __forceinline__ unsigned int float_key(float f) {
  const unsigned int u = __float_as_uint(f);
  if (f != f) return 0xFFFFFFFEu;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(unsigned int k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// Batcher's odd-even merge sort written out comparator by comparator (5 / 19 / 63 compare-exchanges), so that every index
// is a constant and the keys never leave registers
#define CX(i, j) { const unsigned int lo_ = min(k[i], k[j]); k[j] = max(k[i], k[j]); k[i] = lo_; }
template <int N> __device__ __forceinline__ void sort_net(unsigned int (&k)[N]);
template <> __device__ __forceinline__ void sort_net<4>(unsigned int (&k)[4]) {
  CX(0, 1) CX(2, 3) CX(0, 2) CX(1, 3) CX(1, 2)
}
template <> __device__ __forceinline__ void sort_net<8>(unsigned int (&k)[8]) {
  CX(0, 1) CX(2, 3) CX(4, 5) CX(6, 7) CX(0, 2) CX(1, 3) CX(4, 6) CX(5, 7) CX(1, 2) CX(5, 6) CX(0, 4) CX(1, 5) CX(2, 6)
  CX(3, 7) CX(2, 4) CX(3, 5) CX(1, 2) CX(3, 4) CX(5, 6)
}
template <> __device__ __forceinline__ void sort_net<16>(unsigned int (&k)[16]) {
  CX(0, 1) CX(2, 3) CX(4, 5) CX(6, 7) CX(8, 9) CX(10, 11) CX(12, 13) CX(14, 15) CX(0, 2) CX(1, 3) CX(4, 6) CX(5, 7)
  CX(8, 10) CX(9, 11) CX(12, 14) CX(13, 15) CX(1, 2) CX(5, 6) CX(9, 10) CX(13, 14) CX(0, 4) CX(1, 5) CX(2, 6) CX(3, 7)
  CX(8, 12) CX(9, 13) CX(10, 14) CX(11, 15) CX(2, 4) CX(3, 5) CX(10, 12) CX(11, 13) CX(1, 2) CX(3, 4) CX(5, 6)
  CX(9, 10) CX(11, 12) CX(13, 14) CX(0, 8) CX(1, 9) CX(2, 10) CX(3, 11) CX(4, 12) CX(5, 13) CX(6, 14) CX(7, 15)
  CX(4, 8) CX(5, 9) CX(6, 10) CX(7, 11) CX(2, 4) CX(3, 5) CX(6, 8) CX(7, 9) CX(10, 12) CX(11, 13) CX(1, 2) CX(3, 4)
  CX(5, 6) CX(7, 8) CX(9, 10) CX(11, 12) CX(13, 14)
}
#undef CX

// One coordinate of mode 3: sort the K keys (padded to N) and sum the K - 2 trim in the middle in ascending order
template <int N>
__device__ __forceinline__ float trimmed_sum(unsigned int (&k)[N], int K, int trim) {
  sort_net<N>(k);
  float s = 0.f;
#pragma unroll
  for (int r = 0; r < N; ++r)
    if (r >= trim && r < K - trim) s += key_float(k[r]);
  return s;
}

// ---------------------------------------------------------------------------------------------
// Mode 4: Bulyan's coordinate stage (El Mhamdi, Guerraoui and Rouault, ICML 2018).  The K = theta rows named by `select`
// (bulyan_select's choice) are sorted per coordinate as in mode 3.  m is the median in fp32: the middle value for odd K,
// 0.5f * a + 0.5f * b of the two middle values for even K.  The beta = K - 2 trim values nearest to m are a window
// [s, s + beta) of the sorted order with s in [0, 2 trim]: starting from s = 0, the window moves right while the value
// entering it is strictly nearer to m than the value leaving it (distance fabsf(v - m), NaN farthest), or equal to it, so a
// tie in distance keeps the smaller value.  The window is summed in ascending order in fp32 like mode 3.
//
// The entering value sits beta places after the leaving one.  beta is the same for the whole launch, so a barrel shift of
// the sorted keys by beta (one conditional shift per bit of beta) lines them up under constant register indices; the
// median is read the same way, through a shift by (K - 1) / 2 (a plain `r == mid` select loop is turned into an indexed
// load by the compiler and puts the keys in local memory).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool nearer(float d, float e) { return d < e || (e != e && d == d); }   // NaN farthest

// sh[j] <- sh[j + n] for the bits B, 2B, ... <= N of n (padding shifts in past the end); one template level per bit so that
// every index is a constant
template <int N, int B>
__device__ __forceinline__ void barrel_shift(unsigned int (&sh)[N], int n) {
  if constexpr (B <= N) {
    if (n & B) {
#pragma unroll
      for (int j = 0; j < N; ++j) sh[j] = j + B < N ? sh[j + B] : 0xFFFFFFFFu;
    }
    barrel_shift<N, 2 * B>(sh, n);
  }
}

template <int N>
__device__ __forceinline__ float near_median_sum(unsigned int (&k)[N], int K, int trim) {
  const int beta = K - 2 * trim, span = 2 * trim;
  sort_net<N>(k);
  unsigned int md[N];                                          // md[0], md[1] = k[(K - 1) / 2], k[(K - 1) / 2 + 1]
#pragma unroll
  for (int j = 0; j < N; ++j) md[j] = k[j];
  barrel_shift<N, 1>(md, (K - 1) / 2);
  const float lo = key_float(md[0]), hi = key_float(md[1]);
  const float m = (K & 1) ? lo : __fadd_rn(__fmul_rn(0.5f, lo), __fmul_rn(0.5f, hi));
  unsigned int sh[N];                                          // sh[j] = k[j + beta]
#pragma unroll
  for (int j = 0; j < N; ++j) sh[j] = k[j];
  barrel_shift<N, 1>(sh, beta);
  int s = 0;
  bool moving = true;
#pragma unroll
  for (int j = 0; j < N - 1; ++j) {
    if (j < span && moving) {
      const float vin = key_float(sh[j]), vout = key_float(k[j]);
      moving = nearer(fabsf(__fsub_rn(vin, m)), fabsf(__fsub_rn(vout, m))) || vin == vout || (vin != vin && vout != vout);
      s += moving;
    }
  }
  float sum = 0.f;
#pragma unroll
  for (int r = 0; r < N; ++r)
    if (r >= s && r < s + beta) sum += key_float(k[r]);
  return sum;
}

// Modes 3 and 4 on raw rows: the thread loads its 4 coordinates of the K rows as keys (row r of `tensor` is worker slot
// select[r][tensor] with SEL, slot r without), then reduces every coordinate with trimmed_sum or near_median_sum.
template <int MODE, int N, bool SEL>
__device__ __forceinline__ float4 raw_robust_f4(const UpdateArgs& a, long long idx, int tensor) {
  const int K = a.K, trim = a.trim;
  unsigned int k[4][N];
#pragma unroll
  for (int r = 0; r < N; ++r) {
    if (r < a.K) {
      const int slot = SEL ? a.select[r * a.tv.ntensors + tensor] : r;
      const float4 v = ld_f4(reinterpret_cast<const float4*>(a.grad_in + slot * a.slot_stride + idx));
      k[0][r] = float_key(v.x); k[1][r] = float_key(v.y); k[2][r] = float_key(v.z); k[3][r] = float_key(v.w);
    } else {
      k[0][r] = k[1][r] = k[2][r] = k[3][r] = 0xFFFFFFFFu;
    }
  }
  float out[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) out[e] = MODE == 3 ? trimmed_sum<N>(k[e], K, trim) : near_median_sum<N>(k[e], K, trim);
  return make_float4(out[0], out[1], out[2], out[3]);
}

// ---------------------------------------------------------------------------------------------
// Modes 3 and 4 behind nearest-neighbour mixing (MIX; robust.cu nnm_mix_kernel).  The thread loads the mixP raw rows (slots
// 0..mixP-1) once.  Per coordinate, mixed row i is formed in fp32 exactly as
//     y = +0.0f;  for j = 0, 1, ..., mixP - 1 in ascending order: if bit j of mask_i is set, y = y + x_j  (round to nearest);
//     y = y * mix_scale  (one rounded multiply, mix_scale = fp32(1 / n_mix)),
// with mask_i = mix[i][t] for mode 3 (the K = mixP mixed rows) and mask_r = mix[select[r][t]][t] for mode 4 (the K = theta
// mixed rows bulyan_select chose).  The K mixed values are then reduced by trimmed_sum / near_median_sum as in raw_robust_f4.
// The raw rows stay in registers (N = SORT_N >= mixP float4s); the keys are built one coordinate at a time, which holds the
// registers down where raw_robust_f4 keeps the keys of all 4 coordinates.
// ---------------------------------------------------------------------------------------------
template <int MODE, int N>
__device__ __forceinline__ float4 mixed_robust_f4(const UpdateArgs& a, long long idx, int tensor) {
  const int T = a.tv.ntensors;
  float4 x[N];
#pragma unroll
  for (int j = 0; j < N; ++j)
    if (j < a.mixP) x[j] = ld_f4(reinterpret_cast<const float4*>(a.grad_in + j * a.slot_stride + idx));
  unsigned int mask[N];
#pragma unroll
  for (int r = 0; r < N; ++r) mask[r] = r < a.K ? a.mix[(MODE == 4 ? a.select[r * T + tensor] : r) * T + tensor] : 0u;
  float out[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    unsigned int k[N];
#pragma unroll
    for (int r = 0; r < N; ++r) {
      float y = 0.f;
#pragma unroll
      for (int j = 0; j < N; ++j) {
        const float v = e == 0 ? x[j].x : e == 1 ? x[j].y : e == 2 ? x[j].z : x[j].w;
        if (j < a.mixP && ((mask[r] >> j) & 1u)) y = __fadd_rn(y, v);
      }
      k[r] = r < a.K ? float_key(__fmul_rn(y, a.mix_scale)) : 0xFFFFFFFFu;
    }
    out[e] = MODE == 3 ? trimmed_sum<N>(k, a.K, a.trim) : near_median_sum<N>(k, a.K, a.trim);
  }
  return make_float4(out[0], out[1], out[2], out[3]);
}

// ---------------------------------------------------------------------------------------------
// Mode 7: mode 3 over worker-bucket rows (--bucketing; bucketing.cu wbucket_plan_kernel; codes/oracle.py::wbucket_rows).
// Bucket row r holds the raw slots of wb_mask[r].  Per coordinate it is formed in fp32 as
//     y = -0.0f;  for the member slots j in ascending order: y = y + x_j  (round to nearest);  y = y * wb_scale[r]  (rounded),
// where -0.0f + x_j is x_j for every x_j, so y starts from the lowest member; a one-member row is that member (times 1.0f,
// which changes at most a NaN's payload, and every NaN maps to the same key).  The buckets are disjoint, so each raw value is
// loaded once and summed into its own row only; the K = nb row values are then reduced by trimmed_sum as in raw_robust_f4,
// with the network chosen from nb (SORT_N >= K), not from P.
// ---------------------------------------------------------------------------------------------
template <int N>
__device__ __forceinline__ float4 wbucket_robust_f4(const UpdateArgs& a, long long idx) {
  float4 y[N];
#pragma unroll
  for (int r = 0; r < N; ++r) {
    y[r] = make_float4(-0.f, -0.f, -0.f, -0.f);
    if (r < a.K) {
      for (unsigned int m = a.wb_mask[r]; m; m &= m - 1u) {
        const float4 v = ld_f4(reinterpret_cast<const float4*>(a.grad_in + (__ffs(m) - 1) * a.slot_stride + idx));
        y[r].x = __fadd_rn(y[r].x, v.x); y[r].y = __fadd_rn(y[r].y, v.y);
        y[r].z = __fadd_rn(y[r].z, v.z); y[r].w = __fadd_rn(y[r].w, v.w);
      }
      const float sc = a.wb_scale[r];
      y[r].x = __fmul_rn(y[r].x, sc); y[r].y = __fmul_rn(y[r].y, sc);
      y[r].z = __fmul_rn(y[r].z, sc); y[r].w = __fmul_rn(y[r].w, sc);
    }
  }
  float out[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    unsigned int k[N];
#pragma unroll
    for (int r = 0; r < N; ++r) {
      const float v = e == 0 ? y[r].x : e == 1 ? y[r].y : e == 2 ? y[r].z : y[r].w;
      k[r] = r < a.K ? float_key(v) : 0xFFFFFFFFu;
    }
    out[e] = trimmed_sum<N>(k, a.K, a.trim);
  }
  return make_float4(out[0], out[1], out[2], out[3]);
}

// ---------------------------------------------------------------------------------------------
// Mode 5: centered clipping (clip.cu; codes/oracle.py::centered_clip).  Per coordinate, from acc = +0 and for the rows k in
// ascending order whose weight w_k = w[tensor][k] (cc_weights_kernel) is not zero: acc = fma_rn(w_k, rn(x_k - v), acc); then
// g = rn(v + acc), stored back as the next step's centre.  A zero weight (a NaN or +Inf distance) skips the row's load, so
// such a row never reaches g through 0 * NaN.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 centered_clip_f4(const UpdateArgs& a, long long idx, int tensor) {
  const float* wts = reinterpret_cast<const float*>(a.recomb);
  const float4 v = *reinterpret_cast<const float4*>(a.center + idx);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int k = 0; k < a.K; ++k) {
    const float w = wts[tensor * a.K + k];
    if (w == 0.f) continue;
    const int slot = a.select ? a.select[k * a.tv.ntensors + tensor] : k;
    const float4 x = ld_f4(reinterpret_cast<const float4*>(a.grad_in + slot * a.slot_stride + idx));
    acc.x = __fmaf_rn(w, __fsub_rn(x.x, v.x), acc.x); acc.y = __fmaf_rn(w, __fsub_rn(x.y, v.y), acc.y);
    acc.z = __fmaf_rn(w, __fsub_rn(x.z, v.z), acc.z); acc.w = __fmaf_rn(w, __fsub_rn(x.w, v.w), acc.w);
  }
  const float4 g = make_float4(__fadd_rn(v.x, acc.x), __fadd_rn(v.y, acc.y), __fadd_rn(v.z, acc.z), __fadd_rn(v.w, acc.w));
  *reinterpret_cast<float4*>(a.center + idx) = g;
  return g;
}

// Mode 8: mode 5 over the K = nb worker-bucket rows (--bucketing).  Row k, for a non-zero weight only, is formed per coordinate
// as in mode 7 (members ascending from -0.0f, then times wb_scale[k]); a bucket of zero weight is never read.
__device__ __forceinline__ float4 centered_clip_wbucket_f4(const UpdateArgs& a, long long idx, int tensor) {
  const float* wts = reinterpret_cast<const float*>(a.recomb);
  const float4 v = *reinterpret_cast<const float4*>(a.center + idx);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int k = 0; k < a.K; ++k) {
    const float w = wts[tensor * a.K + k];
    if (w == 0.f) continue;
    float4 x = make_float4(-0.f, -0.f, -0.f, -0.f);
    for (unsigned int m = a.wb_mask[k]; m; m &= m - 1u) {
      const float4 y = ld_f4(reinterpret_cast<const float4*>(a.grad_in + (__ffs(m) - 1) * a.slot_stride + idx));
      x.x = __fadd_rn(x.x, y.x); x.y = __fadd_rn(x.y, y.y); x.z = __fadd_rn(x.z, y.z); x.w = __fadd_rn(x.w, y.w);
    }
    const float sc = a.wb_scale[k];
    x.x = __fmul_rn(x.x, sc); x.y = __fmul_rn(x.y, sc); x.z = __fmul_rn(x.z, sc); x.w = __fmul_rn(x.w, sc);
    acc.x = __fmaf_rn(w, __fsub_rn(x.x, v.x), acc.x); acc.y = __fmaf_rn(w, __fsub_rn(x.y, v.y), acc.y);
    acc.z = __fmaf_rn(w, __fsub_rn(x.z, v.z), acc.z); acc.w = __fmaf_rn(w, __fsub_rn(x.w, v.w), acc.w);
  }
  const float4 g = make_float4(__fadd_rn(v.x, acc.x), __fadd_rn(v.y, acc.y), __fadd_rn(v.z, acc.z), __fadd_rn(v.w, acc.w));
  *reinterpret_cast<float4*>(a.center + idx) = g;
  return g;
}

// ---------------------------------------------------------------------------------------------
// Mode 6: signSGD with majority vote (Bernstein et al., ICLR 2019; codes/oracle.py::sign_vote).  The thread's 4 coordinates are
// bits 4(t % 8) .. 4(t % 8) + 3 of word idx / 32 of each of the K rows.  Per row the nibble is spread into 4 byte counters (bit e
// to bit 8e: nibble * 0x00204081 & 0x01010101), so one add counts all 4 coordinates (K <= 32 fits a byte).  With n_neg rows
// saying "-" and K - n_neg saying "+": g = +1 if "+" has the majority, -1 if "-" has it, +0 on a tie and on every padding
// coordinate, whatever its bits say.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned int ld_u32(const unsigned int* p) {   // coherent (data written by peers this step)
  unsigned int v;
  asm volatile("ld.global.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ float4 sign_vote_f4(const UpdateArgs& a, int tile) {
  int tensor;
  const int lane_valid = tile_valid(a.tv, tile, tensor) - (int)threadIdx.x * 4;
  const unsigned int* words = reinterpret_cast<const unsigned int*>(a.grad_in) + (long long)tile * (DRC_TILE / 32) + (threadIdx.x >> 3);
  const unsigned int shift = 4u * (threadIdx.x & 7u);
  unsigned int neg = 0u;                                       // byte e: rows whose bit for coordinate e is 1 ("-")
  for (int k = 0; k < a.K; ++k) neg += (((ld_u32(words + k * a.slot_stride) >> shift) & 0xFu) * 0x00204081u) & 0x01010101u;
  float out[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int n_neg = (int)((neg >> (8 * e)) & 0xFFu), n_pos = a.K - n_neg;
    out[e] = e >= lane_valid ? 0.f : n_pos > n_neg ? 1.f : n_neg > n_pos ? -1.f : 0.f;
  }
  return make_float4(out[0], out[1], out[2], out[3]);
}

// SORT_N: modes 3 and 4, the sorting-network size (4, 8 or 16 >= K, or >= mixP with MIX).  Each size is its own instantiation so
// that a launch pays the registers of its own network (4 x SORT_N keys per thread), not those of the largest one.  SEL: rows come
// through the `select` table (DETOX's winners, Bulyan's choice); mode 3 without a table is its own instantiation, mode 4 always
// has one.  MIX: modes 3 and 4 over nearest-neighbour mixed rows (mixed_robust_f4), instantiated as <3, N, false, true> and
// <4, N, true, true>.
template <int MODE, int SORT_N = 0, bool SEL = false, bool MIX = false>
__global__ void __launch_bounds__(DRC_THREADS) aggregate_update_kernel(const __grid_constant__ UpdateArgs a) {
  const HyperParams hp = *a.hp;
  const unsigned long long step = *a.step_ptr;
  const bool first = (step == a.first_step);
  // Adam: step count t = updates so far + 1; bias corrections folded into the step size like the reference
  float adam_step_size = 0.f;
  // fp32 beta and fp32(1 - beta) with 1 - beta formed in fp64 (HyperParams)
  const float beta1 = (float)hp.beta1, beta2 = (float)hp.beta2;
  const float one_minus_beta1 = (float)(1.0 - hp.beta1), one_minus_beta2 = (float)(1.0 - hp.beta2);
  if (hp.optimizer != 0) {
    const double t = (double)(step - a.first_step + 1);
    const double bc1 = 1.0 - pow(hp.beta1, t), bc2 = 1.0 - pow(hp.beta2, t);
    adam_step_size = (float)((double)hp.lr * sqrt(bc2) / bc1);
  }
  const int tile_end = a.tile_end > 0 ? a.tile_end : a.tv.ntiles;
  for (int tile = a.tile_begin + blockIdx.x; tile < tile_end; tile += gridDim.x) {
    const int tensor = a.tv.tile_tensor[tile];
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    if (MODE == 0) {
      for (int k = 0; k < a.K; ++k) {
        const int slot = a.select ? a.select[k * a.tv.ntensors + tensor] : k;
        float4 v = ld_f4(reinterpret_cast<const float4*>(a.grad_in + slot * a.slot_stride + idx));
        g.x += v.x; g.y += v.y; g.z += v.z; g.w += v.w;
      }
    } else if (MODE == 2) {
      const float* wts = reinterpret_cast<const float*>(a.recomb);    // geometric median: sum_k w[tensor][k] * g_{slot k}
      for (int k = 0; k < a.K; ++k) {
        const float w = wts[tensor * a.K + k];
        const int slot = a.select ? a.select[k * a.tv.ntensors + tensor] : k;
        float4 v = ld_f4(reinterpret_cast<const float4*>(a.grad_in + slot * a.slot_stride + idx));
        g.x = fmaf(w, v.x, g.x); g.y = fmaf(w, v.y, g.y); g.z = fmaf(w, v.z, g.z); g.w = fmaf(w, v.w, g.w);
      }
    } else if constexpr (MIX) {
      g = mixed_robust_f4<MODE, SORT_N>(a, idx, tensor);
    } else if constexpr (MODE == 3 || MODE == 4) {
      g = raw_robust_f4<MODE, SORT_N, SEL>(a, idx, tensor);
    } else if constexpr (MODE == 7) {
      g = wbucket_robust_f4<SORT_N>(a, idx);
    } else if constexpr (MODE == 8) {
      g = centered_clip_wbucket_f4(a, idx, tensor);
    } else if constexpr (MODE == 5) {
      g = centered_clip_f4(a, idx, tensor);
    } else if constexpr (MODE == 6) {
      g = sign_vote_f4(a, tile);
    } else {
      for (int k = 0; k < a.K; ++k) {
        const float2 v = a.recomb[tensor * a.K + k];
        if (v.x == 0.f && v.y == 0.f) continue;             // rows outside the healthy set
        const float4* src = reinterpret_cast<const float4*>(a.grad_in + 2 * (k * a.slot_stride + idx));
        float4 c0 = ld_f4(src), c1 = ld_f4(src + 1);        // (re0,im0,re1,im1) (re2,im2,re3,im3)
        // Re(v c) = fma(v.re, c.re, -rn(v.im c.im)), added to the row sum with one rounding
        g.x = __fadd_rn(g.x, __fmaf_rn(v.x, c0.x, -__fmul_rn(v.y, c0.y)));
        g.y = __fadd_rn(g.y, __fmaf_rn(v.x, c0.z, -__fmul_rn(v.y, c0.w)));
        g.z = __fadd_rn(g.z, __fmaf_rn(v.x, c1.x, -__fmul_rn(v.y, c1.y)));
        g.w = __fadd_rn(g.w, __fmaf_rn(v.x, c1.z, -__fmul_rn(v.y, c1.w)));
      }
    }
    if constexpr (MODE != 5 && MODE != 6 && MODE != 8) { g.x *= a.scale; g.y *= a.scale; g.z *= a.scale; g.w *= a.scale; }
    if (a.grad_out) *reinterpret_cast<float4*>(a.grad_out + idx) = g;

    float4 p = *reinterpret_cast<const float4*>(a.params + idx);
    float4 m = *reinterpret_cast<const float4*>(a.momentum + idx);
    float* gp = &g.x; float* pp = &p.x; float* mp = &m.x;
    if (hp.optimizer == 0) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float d = gp[e];
        if (hp.weight_decay != 0.f) d = fmaf(hp.weight_decay, pp[e], d);
        if (hp.momentum != 0.f) {
          float b = first ? d : fmaf(hp.momentum, mp[e], hp.one_minus_dampening * d);
          mp[e] = b;
          d = hp.nesterov ? fmaf(hp.momentum, b, d) : b;
        }
        pp[e] = fmaf(-hp.lr, d, pp[e]);
      }
    } else {
      float4 v = *reinterpret_cast<const float4*>(a.exp_avg_sq + idx);
      float4 vm = (hp.optimizer == 2) ? *reinterpret_cast<const float4*>(a.max_exp_avg_sq + idx) : v;
      float* vp = &v.x; float* vmp = &vm.x;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float d = gp[e];
        if (hp.weight_decay != 0.f) d = fmaf(hp.weight_decay, pp[e], d);
        mp[e] = fmaf(beta1, mp[e], one_minus_beta1 * d);
        vp[e] = fmaf(beta2, vp[e], one_minus_beta2 * d * d);
        float vv = vp[e];
        if (hp.optimizer == 2) { vmp[e] = fmaxf(vmp[e], vv); vv = vmp[e]; }
        pp[e] = fmaf(-adam_step_size, mp[e] / (sqrtf(vv) + hp.eps), pp[e]);
      }
      *reinterpret_cast<float4*>(a.exp_avg_sq + idx) = v;
      if (hp.optimizer == 2) *reinterpret_cast<float4*>(a.max_exp_avg_sq + idx) = vm;
    }
    *reinterpret_cast<float4*>(a.momentum + idx) = m;
    *reinterpret_cast<float4*>(a.params + idx) = p;
    if (a.mc_params) {
      multimem_st_f4(reinterpret_cast<float4*>(a.mc_params + idx), p);
    } else {
#pragma unroll 1
      for (int d = 0; d < a.ndst; ++d) st_f4(reinterpret_cast<float4*>(a.dst[d] + idx), p);
    }
  }
  if (grid_last_cta(a.done_counter)) {
    if ((int)threadIdx.x < a.flags.n) st_release_sys(a.flags.ptr[threadIdx.x], step + 1);
  }
}

// modes 3 and 4: the instantiation with the smallest sorting network that holds `rows` (K, or mixP with mixing)
template <int MODE, bool SEL, bool MIX>
static void launch_sorted(const UpdateArgs* args, int rows, int grid, cudaStream_t stream) {
  if (rows <= 4) aggregate_update_kernel<MODE, 4, SEL, MIX><<<grid, DRC_THREADS, 0, stream>>>(*args);
  else if (rows <= 8) aggregate_update_kernel<MODE, 8, SEL, MIX><<<grid, DRC_THREADS, 0, stream>>>(*args);
  else aggregate_update_kernel<MODE, 16, SEL, MIX><<<grid, DRC_THREADS, 0, stream>>>(*args);
}

extern "C" int drc_aggregate_update(const UpdateArgs* args, int grid, cudaStream_t stream) {
  const int mode = args->mode, K = args->K;
  if (args->ndst > DRC_MAX_DST || args->flags.n > DRC_MAX_DST) return (int)cudaErrorInvalidValue;
  // modes 3 and 4 sort K <= TRIM_MAXP rows per coordinate and keep K - 2 trim of them; mode 4 reads its K = theta rows
  // through the table bulyan_select filled
  if ((mode == 3 || mode == 4 || mode == 7) && (K < 1 || K > TRIM_MAXP || args->trim < 0 || 2 * args->trim >= K))
    return (int)cudaErrorInvalidValue;
  if (mode == 4 && !args->select) return (int)cudaErrorInvalidValue;
  // centered clipping: K <= TRIM_MAXP rows (through `select` or slots 0..K-1), their weights and the centre
  if (mode == 5) {
    if (K < 1 || K > TRIM_MAXP || !args->recomb || !args->center || args->mix) return (int)cudaErrorInvalidValue;
    aggregate_update_kernel<5><<<grid, DRC_THREADS, 0, stream>>>(*args);
    return (int)cudaGetLastError();
  }
  // worker buckets: the trimmed mean / median of K = nb <= TRIM_MAXP bucket rows, formed from the masks and scales of
  // wbucket_plan_kernel (no row table, no mixing)
  if (mode == 7) {
    if (!args->wb_mask || !args->wb_scale || args->select || args->mix) return (int)cudaErrorInvalidValue;
    launch_sorted<7, false, false>(args, K, grid, stream);
    return (int)cudaGetLastError();
  }
  // centered clipping over the K = nb worker-bucket rows
  if (mode == 8) {
    if (K < 1 || K > TRIM_MAXP || !args->recomb || !args->center || !args->wb_mask || !args->wb_scale || args->select || args->mix)
      return (int)cudaErrorInvalidValue;
    aggregate_update_kernel<8><<<grid, DRC_THREADS, 0, stream>>>(*args);
    return (int)cudaGetLastError();
  }
  // signSGD majority vote: K = P <= 32 sign rows in slots 0..K-1 (the adversary bitmaps' width), no row table
  if (mode == 6) {
    if (K < 1 || K > DRC_MAX_WORKERS || args->select || args->mix) return (int)cudaErrorInvalidValue;
    aggregate_update_kernel<6><<<grid, DRC_THREADS, 0, stream>>>(*args);
    return (int)cudaGetLastError();
  }
  // nearest-neighbour mixing: modes 3 (K = mixP mixed rows, no row table) and 4 (K = theta mixed rows named by `select`)
  if (args->mix) {
    if (args->mixP < 1 || args->mixP > TRIM_MAXP || !(args->mix_scale > 0.f)) return (int)cudaErrorInvalidValue;
    if (mode == 3 && K == args->mixP && !args->select) launch_sorted<3, false, true>(args, args->mixP, grid, stream);
    else if (mode == 4 && K <= args->mixP) launch_sorted<4, true, true>(args, args->mixP, grid, stream);
    else return (int)cudaErrorInvalidValue;
    return (int)cudaGetLastError();
  }
  // a row table names at most TRIM_MAXP rows under the weighted sum (the weight-space geometric median's limit); the cyclic
  // recombination reads every worker's slot and has no use for one
  if (args->select && (mode == 1 || (mode == 2 && (K < 1 || K > TRIM_MAXP)))) return (int)cudaErrorInvalidValue;
  if (mode == 0) aggregate_update_kernel<0><<<grid, DRC_THREADS, 0, stream>>>(*args);
  else if (mode == 2) aggregate_update_kernel<2><<<grid, DRC_THREADS, 0, stream>>>(*args);
  else if (mode == 3 && args->select) launch_sorted<3, true, false>(args, K, grid, stream);
  else if (mode == 3) launch_sorted<3, false, false>(args, K, grid, stream);
  else if (mode == 4) launch_sorted<4, true, false>(args, K, grid, stream);
  else aggregate_update_kernel<1><<<grid, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Worker side: refresh the bf16 compute copy of the matrix-like parameters from the fp32 arena the PS
// just wrote (one streaming pass over the tiles flagged bf16).
// ---------------------------------------------------------------------------------------------
struct CastArgs {
  const float* src;
  __nv_bfloat16* dst;
  TileView tv;
};

__global__ void __launch_bounds__(DRC_THREADS) cast_params_kernel(const __grid_constant__ CastArgs a) {
  for (int tile = blockIdx.x; tile < a.tv.ntiles; tile += gridDim.x) {
    const int tensor = a.tv.tile_tensor[tile];
    if (!a.tv.meta[tensor].is_bf16) continue;
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    float4 v = ld_f4(reinterpret_cast<const float4*>(a.src + idx));
    __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
    uint2 out;
    out.x = *reinterpret_cast<unsigned int*>(&lo);
    out.y = *reinterpret_cast<unsigned int*>(&hi);
    *reinterpret_cast<uint2*>(a.dst + idx) = out;
  }
}

extern "C" int drc_cast_params(const CastArgs* args, int grid, cudaStream_t stream) {
  cast_params_kernel<<<grid, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Flag / step utilities.  Waiters poll flags in their *own* memory; a watchdog turns a lost peer into a
// host-visible error code instead of a silent hang (the reference blocks forever in MPI waitany).
// ---------------------------------------------------------------------------------------------
struct WaitArgs {
  const unsigned long long* flags[DRC_MAX_WORKERS];
  int n;
  const unsigned long long* step_ptr;
  long long addend;               // wait until flag >= *step_ptr + addend
  unsigned long long timeout_ns;  // 0 = wait forever
  int* error;                     // device int: set to 1 + index of the first flag that timed out
  unsigned long long* stamps;     // optional trace ring [64][2]: %globaltimer at entry / at release (the "Comm" time the
                                  // reference prints per step, src/worker/baseline_worker.py:148-150, measured on the device)
};

__global__ void wait_flags_kernel(const __grid_constant__ WaitArgs a) {
  const int i = threadIdx.x;
  const unsigned long long cur = *a.step_ptr;
  unsigned long long t0 = 0;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t0));
  if (i < a.n) {
    const unsigned long long want = cur + a.addend;
    unsigned int backoff = 32;
    while (ld_acquire_sys(a.flags[i]) < want) {
      __nanosleep(backoff);
      if (backoff < 512) backoff <<= 1;
      if (a.timeout_ns) {
        unsigned long long t1;
        asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t1));
        if (t1 - t0 > a.timeout_ns) { atomicCAS(a.error, 0, i + 1); break; }
      }
    }
  }
  __syncwarp();
  if (a.stamps && i == 0) {
    unsigned long long t1;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t1));
    a.stamps[(cur & 63) * 2] = t0;
    a.stamps[(cur & 63) * 2 + 1] = t1;
  }
}

extern "C" int drc_wait_flags(const WaitArgs* args, cudaStream_t stream) {
  if (args->n > DRC_MAX_WORKERS) return (int)cudaErrorInvalidValue;
  wait_flags_kernel<<<1, 32, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}

__global__ void step_add_kernel(unsigned long long* step, long long delta) { *step += delta; }

extern "C" int drc_step_add(unsigned long long* step, long long delta, cudaStream_t stream) {
  step_add_kernel<<<1, 1, 0, stream>>>(step, delta);
  return (int)cudaGetLastError();
}

// Phase stamp: ring[(step & 63) * 8 + col] = %globaltimer.  One thread; placed at phase boundaries of the captured step so that the
// per-step Comp / Comm / Method / Update times the reference prints (src/worker/cyclic_worker.py:154-156, src/master/
// cyclic_master.py:143) exist in graph mode too, measured on the device with no host synchronisation.
__global__ void stamp_kernel(unsigned long long* ring, const unsigned long long* step_ptr, int col) {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  ring[((*step_ptr) & 63ull) * 8ull + (unsigned long long)col] = t;
}

extern "C" int drc_stamp(unsigned long long* ring, const unsigned long long* step_ptr, int col, cudaStream_t stream) {
  stamp_kernel<<<1, 1, 0, stream>>>(ring, step_ptr, col);
  return (int)cudaGetLastError();
}

struct SetFlagArgs {
  FlagList flags;
  const unsigned long long* step_ptr;
  long long addend;
};

__global__ void set_flags_kernel(const __grid_constant__ SetFlagArgs a) {
  if ((int)threadIdx.x < a.flags.n) {
    fence_sys();
    st_release_sys(a.flags.ptr[threadIdx.x], *a.step_ptr + a.addend);
  }
}

extern "C" int drc_set_flags(const SetFlagArgs* args, cudaStream_t stream) {
  set_flags_kernel<<<1, 32, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}

extern "C" int drc_sizeof_UpdateArgs() { return (int)sizeof(UpdateArgs); }
extern "C" int drc_sizeof_CastArgs() { return (int)sizeof(CastArgs); }
extern "C" int drc_sizeof_WaitArgs() { return (int)sizeof(WaitArgs); }
extern "C" int drc_sizeof_SetFlagArgs() { return (int)sizeof(SetFlagArgs); }
extern "C" int drc_sizeof_TensorMeta() { return (int)sizeof(TensorMeta); }
extern "C" int drc_sizeof_HyperParams() { return (int)sizeof(HyperParams); }
extern "C" int drc_sizeof_TileView() { return (int)sizeof(TileView); }
extern "C" int drc_sizeof_FlagList() { return (int)sizeof(FlagList); }
