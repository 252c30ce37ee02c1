// Fused softmax cross-entropy + gradient + Prec@1 / Prec@5 for the classifier head (one launch instead of ~20).
//
// The worker's loss tail -- logits.float(), log_softmax, nll_loss, their two backward kernels, the cast of the gradient
// back to bf16, topk, eq, the reductions and the three scalar updates of the metrics tensor -- is a chain of ~20 dependent
// short launches on a [B, 10] tensor.  This kernel reads the logits once and
// produces everything: mean loss, d(loss)/d(logits) = (softmax - onehot) / B in the logits' dtype, and the Prec@k counts,
// accumulated straight into the worker's metrics tensor (loss, prec1, prec5).  One warp per row, rows distributed over the
// 32 warps of ONE CTA, all cross-row sums folded in a fixed order (bit-deterministic, as the exact-equality vote needs).
//
// Prec@k follows the reference's `accuracy()` (src/worker/utils.py:22-35): a row counts for Prec@k when fewer than k logits
// are strictly greater than the label's logit (ties resolve in favour of the label).
//
// Rows are spread over the 32 warps of one CTA; for C <= 32 (CIFAR / MNIST heads) a row lives in one register per lane and four
// rows per warp are in flight at once, so B = 128 costs a single global round trip.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

struct CeArgs {
  const void* logits;              // [B, C] bf16 or fp32, row pitch = C
  int is_bf16;
  const long long* labels;         // [B]
  void* dlogits;                   // [B, C] same dtype as logits
  float* loss_out;                 // [1] mean loss
  float* metrics;                  // [3] += (loss, prec1 %, prec5 %) * metric_scale   (may be null)
  float metric_scale;
  int B, C;
};

__device__ __forceinline__ float ld_logit(const CeArgs& a, long long i) {
  return a.is_bf16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(a.logits)[i])
                   : reinterpret_cast<const float*>(a.logits)[i];
}

constexpr int CE_WARPS = 32;

// one row, lane-resident logits (C <= 32): everything from registers
__device__ __forceinline__ void ce_row_small(const CeArgs& a, int row, int lane, float z, int label, float inv_b, float& w_loss,
                                             float& w_p1, float& w_p5) {
  const bool act = lane < a.C;
  float mx = act ? z : -3.0e38f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  const float zl = __shfl_sync(0xffffffffu, z, label);
  const float e = act ? __expf(z - mx) : 0.f;
  float se = e;
  int greater = (act && z > zl) ? 1 : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    se += __shfl_xor_sync(0xffffffffu, se, o);
    greater += __shfl_xor_sync(0xffffffffu, greater, o);
  }
  if (act) {
    const float g = (e / se - (lane == label ? 1.f : 0.f)) * inv_b;
    const long long i = (long long)row * a.C + lane;
    if (a.is_bf16) reinterpret_cast<__nv_bfloat16*>(a.dlogits)[i] = __float2bfloat16_rn(g);
    else reinterpret_cast<float*>(a.dlogits)[i] = g;
  }
  w_loss += mx + __logf(se) - zl;
  w_p1 += greater < 1 ? 1.f : 0.f;
  w_p5 += greater < 5 ? 1.f : 0.f;
}

__global__ void __launch_bounds__(CE_WARPS * 32) ce_fused_kernel(const CeArgs a) {
  __shared__ float s_loss[CE_WARPS], s_p1[CE_WARPS], s_p5[CE_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float w_loss = 0.f, w_p1 = 0.f, w_p5 = 0.f;                 // per-warp running sums (every lane holds the same value)
  const float inv_b = 1.0f / (float)a.B;
  if (a.C <= 32) {
    // four rows of a warp in flight at once: one global round trip for B <= 128
    for (int row0 = warp; row0 < a.B; row0 += 4 * CE_WARPS) {
      float z[4]; int lab[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = row0 + i * CE_WARPS;
        z[i] = (row < a.B && lane < a.C) ? ld_logit(a, (long long)row * a.C + lane) : 0.f;
        lab[i] = row < a.B ? (int)a.labels[row] : 0;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = row0 + i * CE_WARPS;
        if (row < a.B) ce_row_small(a, row, lane, z[i], lab[i], inv_b, w_loss, w_p1, w_p5);
      }
    }
  } else {
    for (int row = warp; row < a.B; row += CE_WARPS) {
      const long long base = (long long)row * a.C;
      const int label = (int)a.labels[row];
      float mx = -3.0e38f;
      for (int c = lane; c < a.C; c += 32) mx = fmaxf(mx, ld_logit(a, base + c));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      const float zl = ld_logit(a, base + label);
      float se = 0.f;
      int greater = 0;
      for (int c = lane; c < a.C; c += 32) {
        const float z = ld_logit(a, base + c);
        se += __expf(z - mx);
        greater += (z > zl) ? 1 : 0;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        se += __shfl_xor_sync(0xffffffffu, se, o);
        greater += __shfl_xor_sync(0xffffffffu, greater, o);
      }
      const float lse = mx + __logf(se);
      const float inv_se = 1.0f / se;
      for (int c = lane; c < a.C; c += 32) {
        const float z = ld_logit(a, base + c);
        const float g = (__expf(z - mx) * inv_se - (c == label ? 1.f : 0.f)) * inv_b;
        if (a.is_bf16) reinterpret_cast<__nv_bfloat16*>(a.dlogits)[base + c] = __float2bfloat16_rn(g);
        else reinterpret_cast<float*>(a.dlogits)[base + c] = g;
      }
      w_loss += lse - zl;
      w_p1 += greater < 1 ? 1.f : 0.f;
      w_p5 += greater < 5 ? 1.f : 0.f;
    }
  }
  if (lane == 0) { s_loss[warp] = w_loss; s_p1[warp] = w_p1; s_p5[warp] = w_p5; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float l = 0.f, p1 = 0.f, p5 = 0.f;
    for (int w = 0; w < CE_WARPS; ++w) { l += s_loss[w]; p1 += s_p1[w]; p5 += s_p5[w]; }     // fixed order
    l *= inv_b;
    a.loss_out[0] = l;
    if (a.metrics) {
      a.metrics[0] += l * a.metric_scale;
      a.metrics[1] += p1 * (100.0f * inv_b) * a.metric_scale;
      a.metrics[2] += p5 * (100.0f * inv_b) * a.metric_scale;
    }
  }
}

}  // namespace

extern "C" int drc_ce_fused(const void* logits, int is_bf16, const long long* labels, void* dlogits, float* loss_out, float* metrics,
                            float metric_scale, int B, int C, cudaStream_t stream) {
  if (B < 1 || C < 1) return (int)cudaErrorInvalidValue;
  CeArgs a;
  a.logits = logits; a.is_bf16 = is_bf16; a.labels = labels; a.dlogits = dlogits; a.loss_out = loss_out; a.metrics = metrics;
  a.metric_scale = metric_scale; a.B = B; a.C = C;
  ce_fused_kernel<<<1, CE_WARPS * 32, 0, stream>>>(a);
  return (int)cudaGetLastError();
}
