// Worker buckets (--bucketing s; Karimireddy, He and Jaggi, ICLR 2022; codes/bucketing.py).  One single-thread kernel per step,
// launched before the PS waits for the first gradient bucket: it reads the step from device memory (so graph replays advance
// it with no host involvement), takes row step % len of the permutation schedule, and writes the step's nb = ceil(P / s)
// bucket rows -- bucket b holds perm[b s .. min((b + 1) s, P)) -- as member masks (bit j = slot j) and fp32(1 / |b|) scales,
// rows ordered by their lowest member slot.  The update kernel's mode 7 (aggregate_update.cu) forms the rows from them.
#include "common.cuh"

struct WbucketPlanArgs {
  const int* schedule;            // [len][P] the permutation of slots 0..P-1 of every step
  int len;
  int P;                          // 1 <= P <= 32 (one mask bit per slot)
  int s;                          // bucket size, 1 <= s <= P
  const unsigned long long* step_ptr;
  unsigned int* masks;            // [nb] out
  float* scales;                  // [nb] out
};

__global__ void wbucket_plan_kernel(const __grid_constant__ WbucketPlanArgs a) {
  if (threadIdx.x != 0) return;
  const int* perm = a.schedule + (long long)(*a.step_ptr % (unsigned long long)a.len) * a.P;
  unsigned int bucket_mask[32];                               // by bucket b of the permutation
  const int nb = (a.P + a.s - 1) / a.s;
  for (int b = 0; b < nb; ++b) bucket_mask[b] = 0u;
  for (int i = 0; i < a.P; ++i) bucket_mask[i / a.s] |= 1u << perm[i];
  // rows by lowest member: walk the slots upwards and emit a bucket the first time one of its members comes up
  unsigned int emitted = 0u;
  int r = 0;
  for (int j = 0; j < a.P; ++j) {
    for (int b = 0; b < nb; ++b) {
      if (((bucket_mask[b] >> j) & 1u) && !((emitted >> b) & 1u)) {
        emitted |= 1u << b;
        a.masks[r] = bucket_mask[b];
        a.scales[r] = __fdiv_rn(1.0f, (float)__popc(bucket_mask[b]));
        ++r;
      }
    }
  }
}

extern "C" int drc_wbucket_plan(const WbucketPlanArgs* args, cudaStream_t stream) {
  if (args->P < 1 || args->P > 32 || args->s < 1 || args->s > args->P || args->len < 1) return (int)cudaErrorInvalidValue;
  wbucket_plan_kernel<<<1, 32, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Krum, multi-Krum and the geometric median over the bucket rows.  pair_dist (robust.cu) fills the raw slots' pair table
// (then pair_scope_fold at model scope); wbucket_table_kernel turns it into the nb bucket rows' table, which krum_select /
// geomed_weights read with filled=True; wbucket_fold_kernel turns their choice into weights over the raw slots for update
// mode 2.
//
// Table (codes/oracle.py::wbucket_pair_d2): with c = a_b / |b| - a_k / |k|, ||y_b - y_k||^2 = -1/2 c^T D c = -sum_{i<j} c_i c_j
// D_ij over the members of b and k, summed in fp64 for i, then j, ascending, clamped at 0 (a NaN stays a NaN).  One warp per
// tensor, one lane per bucket pair; the warp then zeroes the raw table, as the selection kernels do with theirs.
// ---------------------------------------------------------------------------------------------
#define WB_MAXP 16
#define WB_THREADS 128

struct WbucketArgs {
  const unsigned int* masks;      // [nb] bucket rows (wbucket_plan_kernel)
  int nb, P, T;
  double* raw_d2;                 // [T][P(P-1)/2] table: read, then zeroed
  double* wb_d2;                  // [T][nb(nb-1)/2] out (table kernel)
  const int* select;              // fold: [m][T] bucket rows chosen (Krum / multi-Krum), or null: use w_rows
  int m;
  const float* w_rows;            // fold: [T][nb] geometric-median weights over the bucket rows
  int* wsel;                      // fold, Krum: [K][T] raw slots, K = min(m s, P)
  float* wts;                     // fold: Krum [T][K] weights of wsel; geometric median [T][P] weights over every slot
  int K;
};

__global__ void __launch_bounds__(WB_THREADS) wbucket_table_kernel(const __grid_constant__ WbucketArgs a) {
  const int tensor = (int)(blockIdx.x * (WB_THREADS / 32) + (threadIdx.x >> 5));
  const int lane = threadIdx.x & 31;
  if (tensor >= a.T) return;                                   // the whole warp leaves together
  const int npr = a.P * (a.P - 1) / 2, npb = a.nb * (a.nb - 1) / 2;
  double* raw = a.raw_d2 + (long long)tensor * npr;
  for (int q = lane; q < npb; q += 32) {
    int k = 1;
    while ((k + 1) * k / 2 <= q) ++k;                          // pair q = (b < k) sits at k (k - 1) / 2 + b
    const int b = q - k * (k - 1) / 2;
    const unsigned int mb = a.masks[b], mk = a.masks[k], u = mb | mk;
    const double cb = __ddiv_rn(1.0, (double)__popc(mb)), ck = -__ddiv_rn(1.0, (double)__popc(mk));
    double acc = 0.0;
    for (unsigned int m1 = u; m1; m1 &= m1 - 1u) {
      const int i = __ffs(m1) - 1;
      const double ci = ((mb >> i) & 1u) ? cb : ck;
      for (unsigned int m2 = u & ~((2u << i) - 1u); m2; m2 &= m2 - 1u) {
        const int j = __ffs(m2) - 1;
        const double cj = ((mb >> j) & 1u) ? cb : ck;
        acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(ci, cj), raw[j * (j - 1) / 2 + i]));
      }
    }
    const double v = -acc;
    a.wb_d2[(long long)tensor * npb + q] = v < 0.0 ? 0.0 : v;
  }
  __syncwarp();
  for (int q = lane; q < npr; q += 32) raw[q] = 0.0;
}

// One thread per tensor.  Each chosen bucket row of weight w_b (1 / m for Krum / multi-Krum, the Weiszfeld weight for the
// geometric median) gives its members w_b / |b|, formed in fp64 and rounded to fp32 once.  Krum / multi-Krum write the compact
// table: the chosen buckets in selection order, members ascending, padded to K entries with weight 0 on the first chosen slot,
// so a slot outside every chosen bucket is never read.  The geometric median writes a weight for every slot.
__global__ void wbucket_fold_kernel(const __grid_constant__ WbucketArgs a) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.T) return;
  if (!a.select) {
    for (int b = 0; b < a.nb; ++b) {
      const unsigned int mb = a.masks[b];
      const float w = (float)__ddiv_rn((double)a.w_rows[t * a.nb + b], (double)__popc(mb));
      for (unsigned int m1 = mb; m1; m1 &= m1 - 1u) a.wts[t * a.P + (__ffs(m1) - 1)] = w;
    }
    return;
  }
  const double wm = __ddiv_rn(1.0, (double)a.m);
  int k = 0, first = -1;
  for (int r = 0; r < a.m; ++r) {
    const unsigned int mb = a.masks[a.select[r * a.T + t]];
    const float w = (float)__ddiv_rn(wm, (double)__popc(mb));
    for (unsigned int m1 = mb; m1 && k < a.K; m1 &= m1 - 1u, ++k) {
      const int j = __ffs(m1) - 1;
      if (first < 0) first = j;
      a.wsel[k * a.T + t] = j;
      a.wts[t * a.K + k] = w;
    }
  }
  for (; k < a.K; ++k) {
    a.wsel[k * a.T + t] = first;
    a.wts[t * a.K + k] = 0.f;
  }
}

extern "C" int drc_wbucket_table(const WbucketArgs* args, cudaStream_t stream) {
  if (args->P < 2 || args->P > WB_MAXP || args->nb < 2 || args->nb > args->P || args->T < 1 || !args->masks || !args->raw_d2 ||
      !args->wb_d2)
    return (int)cudaErrorInvalidValue;
  const int warps = WB_THREADS / 32;
  wbucket_table_kernel<<<(args->T + warps - 1) / warps, WB_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}

extern "C" int drc_wbucket_fold(const WbucketArgs* args, cudaStream_t stream) {
  if (args->P < 1 || args->P > WB_MAXP || args->nb < 1 || args->nb > args->P || args->T < 1 || !args->masks || !args->wts)
    return (int)cudaErrorInvalidValue;
  if (args->select ? (args->m < 1 || args->m > args->nb || !args->wsel || args->K < 1 || args->K > args->P) : !args->w_rows)
    return (int)cudaErrorInvalidValue;
  wbucket_fold_kernel<<<(args->T + 127) / 128, 128, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}

extern "C" int drc_sizeof_WbucketPlanArgs() { return (int)sizeof(WbucketPlanArgs); }
extern "C" int drc_sizeof_WbucketArgs() { return (int)sizeof(WbucketArgs); }
