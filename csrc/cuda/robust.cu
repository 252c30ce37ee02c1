// K5 / K6: robust-aggregation baselines on the PS GPU, per parameter tensor.
//
// Geometric median -- reference: `hd.geomedian(np.array(grads), axis=0)` per tensor (hdmedians' Cython
// Weiszfeld loop; src/master/baseline_master.py:271-276).  Here one streaming kernel per Weiszfeld
// iteration: with weights w_i = 1/||g_i - m|| from the previous iteration it forms m_new = sum w_i g_i /
// sum w_i element-wise *and in the same pass* accumulates ||g_i - m_new||^2 for the next iteration plus
// ||m_new - m||^2 for the stopping rule, so every iteration reads the P x D slab exactly once.  A tiny
// `geomed_prep_kernel` turns the accumulated distances into weights and freezes converged tensors.
//
// The product path does better than one pass per iteration: every Weiszfeld iterate is a convex combination
// m = sum_j w_j g_j of the inputs, and for such a point
//     ||g_i - m||^2 = sum_j w_j D_ij - 1/2 sum_jk w_j w_k D_jk          (D_ij = ||g_i - g_j||^2),
// so the whole iteration lives in the P-dimensional weight space once the P(P-1)/2 pairwise distances are known.
// `pair_dist_kernel` (shared with Krum) reads the slab ONCE, `geomed_weights_kernel` iterates to convergence on one
// warp per tensor in fp64, and the weighted combination is formed inside the fused SGD + broadcast kernel
// (aggregate_update MODE 2): two passes over the P x D slab instead of one per iteration.  The streaming
// per-iteration kernels below remain for P > 16.
//
// Krum -- reference: double Python loop of np.linalg.norm per tensor (baseline_master.py:278-296).  Here one
// pass produces all P(P-1)/2 squared distances per tensor, a one-thread-per-tensor kernel scores and selects,
// and the winner row goes through the fused select + SGD + broadcast kernel.  Multi-Krum (Blanchard et al., NeurIPS 2017)
// selects the m lowest-scoring rows instead, and the same fused kernel averages them.
#include "common.cuh"

#define GM_MAXP DRC_MAX_WORKERS

struct GeoMedArgs {
  const float* grad_in;           // [P][slot_stride]
  long long slot_stride;
  int P;
  TileView tv;
  float* median;                  // [D] current estimate m (in/out)
  const float* weights;           // [T][P]  normalised weights for this iteration
  const int* done;                // [T] tensor converged -> skip
  double* dist2;                  // [T][P] out: ||g_i - m_new||^2 (zero on entry)
  double* move2;                  // [T][2] out: ||m_new - m||^2, ||m_new||^2 (zero on entry)
};

__global__ void __launch_bounds__(DRC_THREADS) geomed_iter_kernel(const __grid_constant__ GeoMedArgs a) {
  __shared__ double s_red[DRC_THREADS / 32];
  for (int tile = blockIdx.x; tile < a.tv.ntiles; tile += gridDim.x) {
    int tensor;
    const int valid = tile_valid(a.tv, tile, tensor);
    if (a.done[tensor]) continue;
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    const bool active = (int)threadIdx.x * 4 < valid;
    float4 m_new = make_float4(0.f, 0.f, 0.f, 0.f), m_old = m_new;
    if (active) {
      m_old = *reinterpret_cast<const float4*>(a.median + idx);
      for (int i = 0; i < a.P; ++i) {
        const float w = a.weights[tensor * a.P + i];
        float4 v = ld_f4(reinterpret_cast<const float4*>(a.grad_in + i * a.slot_stride + idx));
        m_new.x = fmaf(w, v.x, m_new.x); m_new.y = fmaf(w, v.y, m_new.y);
        m_new.z = fmaf(w, v.z, m_new.z); m_new.w = fmaf(w, v.w, m_new.w);
      }
      *reinterpret_cast<float4*>(a.median + idx) = m_new;
    }
    // distances to the new estimate (second read of the slab hits L1/L2: same tile, same CTA)
    for (int i = 0; i <= a.P; ++i) {
      double acc = 0.0;
      if (active) {
        float4 v = (i < a.P) ? ld_f4(reinterpret_cast<const float4*>(a.grad_in + i * a.slot_stride + idx)) : m_old;
        float dx = v.x - m_new.x, dy = v.y - m_new.y, dz = v.z - m_new.z, dw = v.w - m_new.w;
        acc = (double)dx * dx + (double)dy * dy + (double)dz * dz + (double)dw * dw;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
      __syncthreads();
      if (threadIdx.x == 0) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < DRC_THREADS / 32; ++w) s += s_red[w];
        if (i < a.P) atomicAdd(&a.dist2[tensor * a.P + i], s);
        else atomicAdd(&a.move2[tensor * 2], s);
      }
      __syncthreads();
    }
    {
      double acc = active ? (double)m_new.x * m_new.x + (double)m_new.y * m_new.y + (double)m_new.z * m_new.z +
                                (double)m_new.w * m_new.w : 0.0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
      __syncthreads();
      if (threadIdx.x == 0) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < DRC_THREADS / 32; ++w) s += s_red[w];
        atomicAdd(&a.move2[tensor * 2 + 1], s);
      }
      __syncthreads();
    }
  }
}

struct GeoMedPrepArgs {
  int T, P;
  double* dist2;                  // [T][P] consumed and zeroed
  double* move2;                  // [T][2] consumed and zeroed
  float* weights;                 // [T][P] out
  int* done;                      // [T] in/out
  int iter;                       // 0: initialise (weights = 1/P -> first estimate is the mean)
  double eps;                     // relative stopping tolerance
};

__global__ void geomed_prep_kernel(const __grid_constant__ GeoMedPrepArgs a) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.T) return;
  if (a.iter == 0) {
    for (int i = 0; i < a.P; ++i) { a.weights[t * a.P + i] = 1.0f / a.P; a.dist2[t * a.P + i] = 0.0; }
    a.move2[t * 2] = a.move2[t * 2 + 1] = 0.0;
    a.done[t] = 0;
    return;
  }
  if (a.done[t]) return;
  const double mv = a.move2[t * 2], nm = a.move2[t * 2 + 1];
  if (a.iter > 1 && sqrt(mv) <= a.eps * fmax(1.0, sqrt(nm))) a.done[t] = 1;
  double w[GM_MAXP], sum = 0.0;
  bool all_zero = true;
  for (int i = 0; i < a.P; ++i) {
    double d = sqrt(a.dist2[t * a.P + i]);
    w[i] = d > 1e-300 ? 1.0 / d : 0.0;
    all_zero &= !(d > 1e-300);
    sum += w[i];
    a.dist2[t * a.P + i] = 0.0;
  }
  a.move2[t * 2] = a.move2[t * 2 + 1] = 0.0;
  if (all_zero) { a.done[t] = 1; return; }
  for (int i = 0; i < a.P; ++i) a.weights[t * a.P + i] = (float)(w[i] / sum);
}

extern "C" int drc_geomed_iter(const GeoMedArgs* args, int grid, cudaStream_t stream) {
  geomed_iter_kernel<<<grid, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_geomed_prep(const GeoMedPrepArgs* args, cudaStream_t stream) {
  if (args->P > GM_MAXP) return (int)cudaErrorInvalidValue;
  geomed_prep_kernel<<<(args->T + 63) / 64, 64, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Krum
// ---------------------------------------------------------------------------------------------
#define KRUM_MAXP 16
#define KRUM_MAXPAIRS (KRUM_MAXP * (KRUM_MAXP - 1) / 2)
#define KRUM_SELECT_THREADS 64

struct PairDistArgs {
  const float* grad_in;
  long long slot_stride;
  int P;                          // rows compared per tensor
  TileView tv;
  double* pair_d2;                // [T][P*(P-1)/2] zero on entry; pair (i<j) at j*(j-1)/2 + i
  const int* rows;                // [P][T] worker slot of row i for tensor t (DETOX: the vote's winner_slot); null -> slot i
};

__global__ void __launch_bounds__(DRC_THREADS) pair_dist_kernel(const __grid_constant__ PairDistArgs a) {
  __shared__ double s_acc[KRUM_MAXPAIRS];
  const int npairs = a.P * (a.P - 1) / 2;
  for (int tile = blockIdx.x; tile < a.tv.ntiles; tile += gridDim.x) {
    int tensor;
    const int valid = tile_valid(a.tv, tile, tensor);
    for (int q = threadIdx.x; q < npairs; q += DRC_THREADS) s_acc[q] = 0.0;
    __syncthreads();
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    const bool active = (int)threadIdx.x * 4 < valid;
    float4 v[KRUM_MAXP];
#pragma unroll
    for (int i = 0; i < KRUM_MAXP; ++i) {
      if (i < a.P && active) {
        const int slot = a.rows ? a.rows[i * a.tv.ntensors + tensor] : i;
        v[i] = ld_f4(reinterpret_cast<const float4*>(a.grad_in + slot * a.slot_stride + idx));
      }
    }
#pragma unroll
    for (int j = 1; j < KRUM_MAXP; ++j) {
#pragma unroll
      for (int i = 0; i < j; ++i) {
        if (j < a.P) {
          float d = 0.f;
          if (active) {
            float dx = v[i].x - v[j].x, dy = v[i].y - v[j].y, dz = v[i].z - v[j].z, dw = v[i].w - v[j].w;
            d = dx * dx + dy * dy + dz * dz + dw * dw;
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
          if ((threadIdx.x & 31) == 0) atomicAdd(&s_acc[j * (j - 1) / 2 + i], (double)d);   // fp64 from the warp level up
        }
      }
    }
    __syncthreads();
    for (int q = threadIdx.x; q < npairs; q += DRC_THREADS)
      atomicAdd(&a.pair_d2[(long long)tensor * npairs + q], s_acc[q]);
    __syncthreads();
  }
}

// Entry (i, j), i != j, of one tensor's pair table: pair (lo < hi) sits at hi * (hi - 1) / 2 + lo
__device__ __forceinline__ double pair_at(const double* d2, int i, int j) {
  const int lo = i < j ? i : j, hi = i < j ? j : i;
  return d2[hi * (hi - 1) / 2 + lo];
}

struct KrumSelectArgs {
  double* pair_d2;                // consumed and zeroed
  int T, P, s;
  int m;                          // slots selected per tensor: 1 = Krum, P - s = multi-Krum
  int* select;                    // [m][T] the m lowest-scoring worker slots, ordered by (score, index)
  const int* rows;                // [P][T] row -> worker slot (the table pair_dist read) so that `select` holds worker slots;
                                  // null -> row i is slot i
};

// Order of distances and scores: ascending with NaN last (what torch.sort / np.sort do), so that a row that sends NaN gets a
// NaN score and is chosen last, as on the library path; on NaN-free input this is the plain `<`.
__device__ __forceinline__ bool less_nan_last(double x, double y) { return x < y || (y != y && x == x); }

__global__ void krum_select_kernel(const __grid_constant__ KrumSelectArgs a) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.T) return;
  const int npairs = a.P * (a.P - 1) / 2;
  double* d2 = a.pair_d2 + (long long)t * npairs;
  int keep = a.P - a.s - 2;
  if (keep < 0) keep = 0;
  __shared__ double s_score[KRUM_MAXP][KRUM_SELECT_THREADS];
  double* sc = &s_score[0][threadIdx.x];                       // score of slot i at sc[i * KRUM_SELECT_THREADS]
  for (int i = 0; i < a.P; ++i) {
    double nb[KRUM_MAXP]; int c = 0;
    for (int j = 0; j < a.P; ++j) {
      if (j == i) continue;
      nb[c++] = pair_at(d2, i, j);
    }
    for (int x = 1; x < c; ++x) { double k = nb[x]; int y = x - 1; while (y >= 0 && less_nan_last(k, nb[y])) { nb[y + 1] = nb[y]; --y; } nb[y + 1] = k; }
    double score = 0.0;
    for (int x = 0; x < keep && x < c; ++x) score += nb[x];
    sc[i * KRUM_SELECT_THREADS] = score;
  }
  // m rounds of selection among the slots not chosen yet: the first one in index order, replaced by any later one with a
  // strictly lower score (NaN last) -- ties go to the lower index, and m = 1 is the Krum winner
  unsigned int used = 0;
  for (int q = 0; q < a.m; ++q) {
    double best = 0.0; int best_i = -1;
    for (int i = 0; i < a.P; ++i) {
      if ((used >> i) & 1u) continue;
      const double s = sc[i * KRUM_SELECT_THREADS];
      if (best_i < 0 || less_nan_last(s, best)) { best = s; best_i = i; }
    }
    used |= 1u << best_i;
    a.select[q * a.T + t] = a.rows ? a.rows[best_i * a.T + t] : best_i;
  }
  for (int q = 0; q < npairs; ++q) d2[q] = 0.0;
}

// ---------------------------------------------------------------------------------------------
// Bulyan (El Mhamdi, Guerraoui and Rouault, ICML 2018), selection stage: theta = P - 2f rounds of Krum, each moving the
// lowest-scoring row of the remaining set R into the selection.  In a round every row i of R scores the sum of its
// keep = max(|R| - f - 2, 0) smallest squared distances to the other rows of R (ascending, NaN last; zero terms sum to 0),
// and the lowest score wins (NaN last, ties to the lower row).  The coordinate stage is aggregate_update MODE 4.
//
// One warp per tensor, lane i owns row i: it sorts its P - 1 neighbour distances once, with the neighbour's row index
// alongside, in a compare-exchange network with constant indices.  A round then sums the first `keep` entries whose row is
// still in R, and a warp argmin picks the winner.  Nothing is re-sorted, and every array index is a compile-time constant.
// ---------------------------------------------------------------------------------------------
#define BULYAN_SELECT_THREADS 128

struct BulyanSelectArgs {
  double* pair_d2;                // [T][P(P-1)/2] consumed and zeroed
  int T, P, f;                    // P >= 4f + 3 rows, f tolerated
  int* select;                    // [P - 2f][T] out: the worker slot chosen in round k at select[k][t]
  const int* rows;                // [P][T] row -> worker slot (the table pair_dist read); null -> row i is slot i
};

// Distances are sums of squares (>= +0) or NaN, so their bit patterns as unsigned integers order them with NaN last once
// every NaN is made the canonical positive one; ~0 pads the entries past the P - 1 neighbours.
__device__ __forceinline__ unsigned long long dist_key(double d) {
  return d != d ? 0x7FF8000000000000ull : (unsigned long long)__double_as_longlong(d);
}

// Batcher's odd-even merge sort of 16 (key, row) pairs (the 63 comparators of aggregate_update.cu's sort_net<16>), written
// out so that every index is a constant and the pairs never leave registers
#define CXP(x, y) {                                                                                  \
    const bool sw_ = key[y] < key[x];                                                                \
    const unsigned long long kx_ = sw_ ? key[y] : key[x], ky_ = sw_ ? key[x] : key[y];               \
    const int ix_ = sw_ ? id[y] : id[x], iy_ = sw_ ? id[x] : id[y];                                  \
    key[x] = kx_; key[y] = ky_; id[x] = ix_; id[y] = iy_; }
__device__ __forceinline__ void sort_pairs16(unsigned long long (&key)[KRUM_MAXP], int (&id)[KRUM_MAXP]) {
  CXP(0, 1) CXP(2, 3) CXP(4, 5) CXP(6, 7) CXP(8, 9) CXP(10, 11) CXP(12, 13) CXP(14, 15) CXP(0, 2) CXP(1, 3) CXP(4, 6)
  CXP(5, 7) CXP(8, 10) CXP(9, 11) CXP(12, 14) CXP(13, 15) CXP(1, 2) CXP(5, 6) CXP(9, 10) CXP(13, 14) CXP(0, 4) CXP(1, 5)
  CXP(2, 6) CXP(3, 7) CXP(8, 12) CXP(9, 13) CXP(10, 14) CXP(11, 15) CXP(2, 4) CXP(3, 5) CXP(10, 12) CXP(11, 13) CXP(1, 2)
  CXP(3, 4) CXP(5, 6) CXP(9, 10) CXP(11, 12) CXP(13, 14) CXP(0, 8) CXP(1, 9) CXP(2, 10) CXP(3, 11) CXP(4, 12) CXP(5, 13)
  CXP(6, 14) CXP(7, 15) CXP(4, 8) CXP(5, 9) CXP(6, 10) CXP(7, 11) CXP(2, 4) CXP(3, 5) CXP(6, 8) CXP(7, 9) CXP(10, 12)
  CXP(11, 13) CXP(1, 2) CXP(3, 4) CXP(5, 6) CXP(7, 8) CXP(9, 10) CXP(11, 12) CXP(13, 14)
}
#undef CXP

__global__ void __launch_bounds__(BULYAN_SELECT_THREADS) bulyan_select_kernel(const __grid_constant__ BulyanSelectArgs a) {
  const int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= a.T) return;                                        // whole warps: t is uniform across the warp
  const int npairs = a.P * (a.P - 1) / 2;
  double* d2 = a.pair_d2 + (long long)t * npairs;
  unsigned long long key[KRUM_MAXP];
  int id[KRUM_MAXP];
#pragma unroll
  for (int j = 0; j < KRUM_MAXP; ++j) {
    key[j] = ~0ull;
    id[j] = lane;
    if (j < a.P && lane < a.P && j != lane) {
      key[j] = dist_key(pair_at(d2, lane, j));
      id[j] = j;
    }
  }
  __syncwarp();
  for (int q = lane; q < npairs; q += 32) d2[q] = 0.0;
  sort_pairs16(key, id);                                       // the P - 1 neighbours first, nearest first, NaN last

  const int theta = a.P - 2 * a.f;
  unsigned int chosen = 0;                                     // rows moved out of R so far (the same in every lane)
  for (int q = 0; q < theta; ++q) {
    int keep = a.P - q - a.f - 2;                              // |R| = P - q
    if (keep < 0) keep = 0;
    double score = 0.0;
    int n = 0;
#pragma unroll
    for (int x = 0; x < KRUM_MAXP - 1; ++x) {
      if (x < a.P - 1 && !((chosen >> id[x]) & 1u) && n < keep) {
        score += __longlong_as_double((long long)key[x]);
        ++n;
      }
    }
    // warp argmin over the rows still in R: NaN scores last, ties to the lower row
    bool valid = lane < a.P && !((chosen >> lane) & 1u);
    int best = lane;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double s2 = __shfl_xor_sync(0xffffffffu, score, o);
      const int b2 = __shfl_xor_sync(0xffffffffu, best, o);
      const bool v2 = __shfl_xor_sync(0xffffffffu, (int)valid, o) != 0;
      const bool take = v2 && (!valid || less_nan_last(s2, score) || (!less_nan_last(score, s2) && b2 < best));
      if (take) { score = s2; best = b2; valid = true; }
    }
    chosen |= 1u << best;
    if (lane == 0) a.select[q * a.T + t] = a.rows ? a.rows[best * a.T + t] : best;
  }
}

// ---------------------------------------------------------------------------------------------
// Nearest-neighbour mixing (Allouah, Farhadkhani, Guerraoui, Gupta, Pinot and Stephan, AISTATS 2023), per tensor: with
// n_mix = P - f, mixed row y_i is the mean of the rows of N_i = {i} + the n_mix - 1 rows nearest to row i (squared distance,
// ascending, NaN last, ties to the lower row; row i itself comes first even when another row duplicates it).
//
// nnm_mix_kernel: one warp per tensor, lane i owns row i.  It sorts row i's P - 1 neighbour distances with sort_pairs16,
// takes the (n_mix - 1)-th key as a threshold and keeps every neighbour below it plus, among the neighbours equal to it, the
// lowest rows (the network is not stable, so ties are resolved on the row index, not on the sorted position).  The bitmask
// of N_i goes to mix[i][t].  Every mixed row is a fixed combination y = A x / n_mix of the raw rows, so for
// c = (a_i - a_k) / n_mix (which sums to 0), ||y_i - y_k||^2 = -1/2 c^T D c with D the raw table: with u_i = D a_i (lane i
// gathers the rows D[j] of its neighbours through shuffles), S_i = a_i^T u_i and Q_ik = a_k^T u_i,
//     ||y_i - y_k||^2 = (2 Q_ik - S_i - S_k) / (2 n_mix^2),
// in fp64 and clamped at 0 (a NaN stays NaN).  With `mixed_out` the kernel overwrites the raw table with the mixed one for
// krum_select / bulyan_select / geomed_weights, which consume and zero it as usual; without, it zeroes the table (the
// coordinate rules need only the masks).  O(P^3) fp64 work per tensor, no pass over the slab.
// ---------------------------------------------------------------------------------------------
#define NNM_THREADS 128

struct NnmMixArgs {
  double* pair_d2;                // [T][P(P-1)/2] in: raw squared distances; out: the mixed table (mixed_out) or zeros
  int T, P, f;                    // n_mix = P - f rows per neighbourhood, 0 <= f < P <= KRUM_MAXP
  unsigned int* mix;              // [P][T] out: bit j of mix[i][t] = row j is in N_i
  int mixed_out;                  // 1: write the mixed table; 0: zero the table
};

__global__ void __launch_bounds__(NNM_THREADS) nnm_mix_kernel(const __grid_constant__ NnmMixArgs a) {
  const int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= a.T) return;                                        // whole warps: t is uniform across the warp
  const int npairs = a.P * (a.P - 1) / 2;
  double* d2 = a.pair_d2 + (long long)t * npairs;
  unsigned long long key[KRUM_MAXP];
  int id[KRUM_MAXP];
#pragma unroll
  for (int j = 0; j < KRUM_MAXP; ++j) {
    key[j] = ~0ull;                                            // self and padding sort after every neighbour
    id[j] = j;
    if (j < a.P && lane < a.P && j != lane) key[j] = dist_key(pair_at(d2, lane, j));
  }
  sort_pairs16(key, id);                                       // the P - 1 neighbours first, nearest first, NaN last
  const int need = a.P - a.f - 1;                              // neighbours besides row i itself
  unsigned long long thr = 0;                                  // key of the need-th nearest neighbour
#pragma unroll
  for (int x = 0; x < KRUM_MAXP - 1; ++x) if (x < need) thr = key[x];
  int below = 0;
#pragma unroll
  for (int x = 0; x < KRUM_MAXP - 1; ++x) below += x < need && key[x] < thr;
  unsigned int mask = 1u << lane;
#pragma unroll
  for (int x = 0; x < KRUM_MAXP - 1; ++x) {
    int lower_ties = 0;                                        // neighbours with the threshold key and a lower row index
#pragma unroll
    for (int y = 0; y < KRUM_MAXP - 1; ++y) lower_ties += key[y] == thr && id[y] < id[x];
    const bool in = need > 0 && (key[x] < thr || (key[x] == thr && lower_ties < need - below));
    if (in) mask |= 1u << id[x];
  }
  if (lane >= a.P) mask = 0;
  if (lane < a.P) a.mix[lane * a.T + t] = mask;

  if (a.mixed_out) {
    double row[KRUM_MAXP];                                     // row[l] = D[lane][l] (0 on the diagonal and past P)
#pragma unroll
    for (int l = 0; l < KRUM_MAXP; ++l) {
      row[l] = 0.0;
      if (l < a.P && lane < a.P && l != lane) row[l] = pair_at(d2, lane, l);
    }
    __syncwarp();                                              // every lane has read its row before any lane writes
    double u[KRUM_MAXP];                                       // u[l] = sum over j in N_lane of D[j][l]
#pragma unroll
    for (int l = 0; l < KRUM_MAXP; ++l) u[l] = 0.0;
#pragma unroll
    for (int j = 0; j < KRUM_MAXP; ++j) {
      if (j < a.P) {
        const bool nb = (mask >> j) & 1u;
#pragma unroll
        for (int l = 0; l < KRUM_MAXP; ++l) {
          const double v = __shfl_sync(0xffffffffu, row[l], j);
          if (nb && l < a.P) u[l] += v;
        }
      }
    }
    double self = 0.0;                                         // S_lane = a_lane^T D a_lane
#pragma unroll
    for (int l = 0; l < KRUM_MAXP; ++l) if ((mask >> l) & 1u) self += u[l];
    const double inv = 1.0 / (2.0 * (double)(a.P - a.f) * (double)(a.P - a.f));
#pragma unroll
    for (int k = 1; k < KRUM_MAXP; ++k) {
      const unsigned int mk = __shfl_sync(0xffffffffu, mask, k);
      const double sk = __shfl_sync(0xffffffffu, self, k);
      double q = 0.0;                                          // Q_lane,k = a_k^T D a_lane
#pragma unroll
      for (int l = 0; l < KRUM_MAXP; ++l) if ((mk >> l) & 1u) q += u[l];
      if (lane < k && k < a.P) {
        double v = (2.0 * q - self - sk) * inv;
        if (v < 0.0) v = 0.0;                                  // cancellation; a NaN fails the test and stays NaN
        d2[k * (k - 1) / 2 + lane] = v;
      }
    }
  } else {
    __syncwarp();
    for (int q = lane; q < npairs; q += 32) d2[q] = 0.0;
  }
}

// nnm_fold_kernel: a choice made over the mixed rows, as weights over the raw rows: w_raw[t][j] = (1 / n_mix) sum over i with
// j in N_i of w_mix[i], summed in fp64.  w_mix is 1/m on the m mixed rows `select` names (Krum m = 1, multi-Krum m = P - f),
// or the fp32 weights [T][P] of geomed_weights.  aggregate_update MODE 2 (K = P, no row table) then applies w_raw.
struct NnmFoldArgs {
  const unsigned int* mix;        // [P][T] neighbour masks from nnm_mix_kernel
  int T, P, f;
  const int* select;              // [m][T] mixed rows chosen (uniform weight 1/m), or null: use w_mix
  int m;
  const float* w_mix;             // [T][P] weights over the mixed rows (select == null)
  float* w_raw;                   // [T][P] out
};

__global__ void nnm_fold_kernel(const __grid_constant__ NnmFoldArgs a) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= a.T * a.P) return;
  const int t = g / a.P, j = g - t * a.P;
  double acc = 0.0;
  if (a.select) {
    const double w = 1.0 / a.m;
    for (int r = 0; r < a.m; ++r)
      if ((a.mix[a.select[r * a.T + t] * a.T + t] >> j) & 1u) acc += w;
  } else {
    for (int i = 0; i < a.P; ++i)
      if ((a.mix[i * a.T + t] >> j) & 1u) acc += (double)a.w_mix[t * a.P + i];
  }
  a.w_raw[t * a.P + j] = (float)(acc / (double)(a.P - a.f));
}

extern "C" int drc_nnm_mix(const NnmMixArgs* args, cudaStream_t stream) {
  if (args->P < 1 || args->P > KRUM_MAXP || args->f < 0 || args->f >= args->P || !args->mix || !args->pair_d2)
    return (int)cudaErrorInvalidValue;
  nnm_mix_kernel<<<(args->T * 32 + NNM_THREADS - 1) / NNM_THREADS, NNM_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_nnm_fold(const NnmFoldArgs* args, cudaStream_t stream) {
  if (args->P < 1 || args->P > KRUM_MAXP || args->f < 0 || args->f >= args->P || !args->mix || !args->w_raw)
    return (int)cudaErrorInvalidValue;
  if (args->select ? (args->m < 1 || args->m > args->P) : !args->w_mix) return (int)cudaErrorInvalidValue;
  nnm_fold_kernel<<<(args->T * args->P + 127) / 128, 128, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Model scope (--rule-scope model): a squared distance over the whole model is the sum of the per-tensor squared distances.
// pair_scope_fold_kernel sums every pair's T entries in ascending tensor order (fp64; a NaN or Inf in one tensor reaches the
// sum) and writes the sum back into every tensor's table, so krum_select / bulyan_select / geomed_weights / nnm_mix run
// unchanged and make the same choice in every tensor.  One thread per pair, one CTA: P(P-1)/2 <= 120 pairs.  The loads of a
// batch of SCOPE_FOLD tensors are issued together and the sum stays in order.
// ---------------------------------------------------------------------------------------------
#define SCOPE_FOLD 16
__global__ void __launch_bounds__(KRUM_MAXPAIRS) pair_scope_fold_kernel(double* pair_d2, int T, int npairs) {
  const int q = threadIdx.x;
  if (q >= npairs) return;
  double s = 0.0;
  int t = 0;
  for (; t + SCOPE_FOLD <= T; t += SCOPE_FOLD) {
    double b[SCOPE_FOLD];
#pragma unroll
    for (int k = 0; k < SCOPE_FOLD; ++k) b[k] = pair_d2[(long long)(t + k) * npairs + q];
#pragma unroll
    for (int k = 0; k < SCOPE_FOLD; ++k) s = __dadd_rn(s, b[k]);
  }
  for (; t < T; ++t) s = __dadd_rn(s, pair_d2[(long long)t * npairs + q]);
  for (t = 0; t < T; ++t) pair_d2[(long long)t * npairs + q] = s;
}

extern "C" int drc_pair_scope_fold(double* pair_d2, int T, int P, cudaStream_t stream) {
  if (!pair_d2 || T < 1 || P < 2 || P > KRUM_MAXP) return (int)cudaErrorInvalidValue;
  pair_scope_fold_kernel<<<1, KRUM_MAXPAIRS, 0, stream>>>(pair_d2, T, P * (P - 1) / 2);
  return (int)cudaGetLastError();
}

extern "C" int drc_pair_dist(const PairDistArgs* args, int grid, cudaStream_t stream) {
  // with or without a row table: at most KRUM_MAXP rows (the pair table of one tensor lives in shared memory)
  if (args->P > KRUM_MAXP) return (int)cudaErrorInvalidValue;
  pair_dist_kernel<<<grid, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_krum_select(const KrumSelectArgs* args, cudaStream_t stream) {
  if (args->P > KRUM_MAXP || args->m < 1 || args->m > args->P) return (int)cudaErrorInvalidValue;
  krum_select_kernel<<<(args->T + KRUM_SELECT_THREADS - 1) / KRUM_SELECT_THREADS, KRUM_SELECT_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_bulyan_select(const BulyanSelectArgs* args, cudaStream_t stream) {
  if (args->P > KRUM_MAXP || args->f < 0 || args->P < 4 * args->f + 3 || !args->select) return (int)cudaErrorInvalidValue;
  bulyan_select_kernel<<<(args->T * 32 + BULYAN_SELECT_THREADS - 1) / BULYAN_SELECT_THREADS, BULYAN_SELECT_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}


// ---------------------------------------------------------------------------------------------
// Weiszfeld in weight space (one warp per tensor, lane i owns input i; fp64)
// ---------------------------------------------------------------------------------------------
struct GeoMedWeightsArgs {
  double* pair_d2;                // [T][P(P-1)/2] consumed and zeroed
  int T, P, max_iter;
  double eps;                     // stop when no weight moved by more than eps
  float* weights;                 // [T][P] out, sum to 1
  int* iters;                     // [T] out (optional): iterations used
};

__global__ void geomed_weights_kernel(const __grid_constant__ GeoMedWeightsArgs a) {
  const int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= a.T) return;
  const int npairs = a.P * (a.P - 1) / 2;
  double* d2 = a.pair_d2 + (long long)t * npairs;
  double row[KRUM_MAXP];
  double maxd = 0.0;
#pragma unroll
  for (int j = 0; j < KRUM_MAXP; ++j) {
    row[j] = 0.0;
    if (j < a.P && lane < a.P && j != lane) {
      row[j] = pair_at(d2, lane, j);
      maxd = fmax(maxd, row[j]);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) maxd = fmax(maxd, __shfl_xor_sync(0xffffffffu, maxd, o));
  __syncwarp();
  for (int q = lane; q < npairs; q += 32) d2[q] = 0.0;
  double w = lane < a.P ? 1.0 / a.P : 0.0;            // first estimate: the mean
  int it = 0;
  if (maxd > 0.0) {
    const double floor_d = 1e-12 * sqrt(maxd) + 1e-300;
    for (; it < a.max_iter; ++it) {
      double s = 0.0;
#pragma unroll
      for (int j = 0; j < KRUM_MAXP; ++j)
        if (j < a.P) s = fma(__shfl_sync(0xffffffffu, w, j), row[j], s);
      double q = w * s;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      const double dist = fmax(sqrt(fmax(s - 0.5 * q, 0.0)), floor_d);
      double wn = lane < a.P ? 1.0 / dist : 0.0;
      double sum = wn;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      wn /= sum;
      double delta = fabs(wn - w);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) delta = fmax(delta, __shfl_xor_sync(0xffffffffu, delta, o));
      w = wn;
      if (delta <= a.eps) { ++it; break; }
    }
  }
  if (lane < a.P) a.weights[t * a.P + lane] = (float)w;
  if (a.iters && lane == 0) a.iters[t] = it;
}

extern "C" int drc_geomed_weights(const GeoMedWeightsArgs* args, cudaStream_t stream) {
  if (args->P > KRUM_MAXP) return (int)cudaErrorInvalidValue;
  geomed_weights_kernel<<<(args->T * 32 + 127) / 128, 128, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}
extern "C" int drc_sizeof_GeoMedWeightsArgs() { return (int)sizeof(GeoMedWeightsArgs); }

extern "C" int drc_sizeof_GeoMedArgs() { return (int)sizeof(GeoMedArgs); }
extern "C" int drc_sizeof_GeoMedPrepArgs() { return (int)sizeof(GeoMedPrepArgs); }
extern "C" int drc_sizeof_PairDistArgs() { return (int)sizeof(PairDistArgs); }
extern "C" int drc_sizeof_KrumSelectArgs() { return (int)sizeof(KrumSelectArgs); }
extern "C" int drc_sizeof_BulyanSelectArgs() { return (int)sizeof(BulyanSelectArgs); }
extern "C" int drc_sizeof_NnmMixArgs() { return (int)sizeof(NnmMixArgs); }
extern "C" int drc_sizeof_NnmFoldArgs() { return (int)sizeof(NnmFoldArgs); }
