// K1 / K2 / K11: fused worker-side gradient encode + adversary hook + push into the PS's HBM over NVLink.
//
// What it replaces in the reference: per-tensor `astype(float64)` -> `err_simulation` -> `blosc.pack_array`
// -> `comm.isend` (src/worker/baseline_worker.py:258-273, src/worker/rep_worker.py:157-177) and, for the
// cyclic code, the per-layer complex linear combination `sum_k W[rank,k] g_k` (src/worker/cyclic_worker.py:
// 165-194).  Here one kernel streams the flat gradient arena(s) once, applies the encode and the Byzantine
// hook in registers and writes 16-byte words straight into slot `worker` of the PS's `grad_in` arena through
// a peer-mapped pointer; the last CTA publishes a step-stamped release flag in PS memory.  No NCCL / host
// involvement on this path.
#include "common.cuh"

struct PushArgs {
  const float* g32[DRC_MAX_R];            // fp32 gradient arena per input stream (sub-batch)
  const __nv_bfloat16* g16[DRC_MAX_R];    // bf16 gradient arena per input stream
  float coef_re[DRC_MAX_R];               // cyclic encode coefficients W[worker, batch_k]
  float coef_im[DRC_MAX_R];
  int R;                                  // number of input streams (1 unless cyclic)
  int cyclic;                             // 0: dst is float[D]; 1: dst is float2[D] (complex64, interleaved)
  float* dst;                             // peer pointer: this worker's slot in the PS grad_in arena
  TileView tv;
  const unsigned int* adv_bitmap;         // [adv_len] adversary bitmap per step (bit w = worker w lies)
  int adv_len;
  const unsigned long long* step_ptr;     // device step counter (graph-replay safe)
  int worker;                             // 0-based worker slot
  int attack;                             // ATTACK_* (codes/adversary.py)
  float magnitude;                        // -100 in the reference
  unsigned long long seed;
  unsigned int* done_counter;             // local, zero
  unsigned long long* flag;               // peer pointer: PS-side grad_ready[worker]
  float* local_copy;                      // optional local fp32 copy of what was sent (debug / NCCL path), may be null
  int tile_begin, tile_end;               // bucket of tiles to push (tile_end == 0: up to the end of the arena)
  // Zero-copy mode: instead of arenas, a device table [R][ntensors] of pointers to each parameter's gradient tensor
  // exactly where autograd left it (bf16 or fp32 per TensorMeta.is_bf16).  No gather / accumulate pass exists at all.
  const void* const* src_table;
  // Worker-side momentum (push_encode_wmom_kernel only): this worker's fp32 state arena, in the slot's element layout.  Each
  // pushed element becomes m' = rn(rn(wm_beta * m) + rn(wm_scale * g)) (wm_beta = fp32(beta), wm_scale = fp32(1 - beta)),
  // m' is stored back, and the adversary hook acts on a copy of m': a liar's state always follows its true gradient.
  float* wmom;
  float wm_beta;
  float wm_scale;
  // signSGD wire (push_encode_sign*_kernel; appended): dst / local_copy are uint32 words, word w = elements 32w..32w+31 of the
  // slot's element layout, bit b (LSB = 0) = 1 iff element 32w + b is < 0 after momentum and the adversary hook; padding bits 0
  int sign;
};

// counter-based normal generator (Philox-lite: 2 rounds of a 64-bit mix, Box-Muller) keyed by (seed, step, worker, idx)
__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
  return x;
}
__device__ __forceinline__ float2 normal_pair(unsigned long long key, unsigned long long idx) {
  unsigned long long h = mix64(key ^ mix64(idx + 0x9e3779b97f4a7c15ULL));
  float u1 = ((unsigned int)(h >> 40) + 1.0f) * (1.0f / 16777217.0f);   // (0,1]
  float u2 = (unsigned int)(h & 0xffffff) * (1.0f / 16777216.0f);
  float r = sqrtf(-2.0f * __logf(u1));
  float s, c;
  __sincosf(6.28318530718f * u2, &s, &c);
  return make_float2(r * c, r * s);
}

__device__ __forceinline__ float4 load_grad4(const PushArgs& a, int k, int tensor, int is_bf16, long long idx, int lane_valid) {
  if (a.src_table) {
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane_valid <= 0) return g;
    const long long e = idx - a.tv.meta[tensor].offset;          // element index inside the tensor (multiple of 4)
    const void* base = a.src_table[k * a.tv.ntensors + tensor];
    if (is_bf16) g = bf16x4_to_f4(*reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(base) + e));
    else g = ld_stream_f4(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + e));
    if (lane_valid < 4) {                                       // tail of the tensor: lanes past numel read allocator slack
      if (lane_valid < 2) g.y = 0.f;
      if (lane_valid < 3) g.z = 0.f;
      g.w = 0.f;
    }
    return g;
  }
  if (is_bf16) {
    uint2 raw = *reinterpret_cast<const uint2*>(a.g16[k] + idx);
    return bf16x4_to_f4(raw);
  }
  return ld_stream_f4(reinterpret_cast<const float4*>(a.g32[k] + idx));
}

// The value a non-cyclic push sends for the thread's 4 elements: the gradient, advanced into the worker's momentum with WMOM,
// then through the adversary hook
template <bool WMOM>
__device__ __forceinline__ float4 push_value(const PushArgs& a, bool lie, unsigned long long key, int tensor, int is_bf16,
                                             long long idx, int lane_valid) {
  float4 g = load_grad4(a, 0, tensor, is_bf16, idx, lane_valid);
  if constexpr (WMOM) {
    // no FMA: the library-op PS and the oracle (codes/oracle.py worker_momentum) round the two products separately
    float4* mp = reinterpret_cast<float4*>(a.wmom + idx);
    float4 m = *mp;
    m.x = __fadd_rn(__fmul_rn(a.wm_beta, m.x), __fmul_rn(a.wm_scale, g.x));
    m.y = __fadd_rn(__fmul_rn(a.wm_beta, m.y), __fmul_rn(a.wm_scale, g.y));
    m.z = __fadd_rn(__fmul_rn(a.wm_beta, m.z), __fmul_rn(a.wm_scale, g.z));
    m.w = __fadd_rn(__fmul_rn(a.wm_beta, m.w), __fmul_rn(a.wm_scale, g.w));
    *mp = m;
    g = m;
  }
  if (lie) {
    if (a.attack == 1) { g.x *= a.magnitude; g.y *= a.magnitude; g.z *= a.magnitude; g.w *= a.magnitude; }
    else if (a.attack == 2) { g = make_float4(a.magnitude, a.magnitude, a.magnitude, a.magnitude); }
    else if (a.attack == 3) {
      float2 n0 = normal_pair(key, (unsigned long long)idx), n1 = normal_pair(key, (unsigned long long)idx + 2);
      float m = fabsf(a.magnitude);
      g = make_float4(m * n0.x, m * n0.y, m * n1.x, m * n1.y);
    }
    // padding must stay zero so that per-tensor rules never see it
    if (lane_valid < 4) {
      if (lane_valid < 1) g.x = 0.f;
      if (lane_valid < 2) g.y = 0.f;
      if (lane_valid < 3) g.z = 0.f;
      g.w = 0.f;
    }
  }
  return g;
}

// The tile loop of the push; returns the step it pushed.  WMOM: the worker-momentum build.  SIGN: the signSGD build, which
// sends one bit per element (PushArgs::sign).
template <bool WMOM, bool SIGN = false>
__device__ __forceinline__ unsigned long long push_encode_tiles(const PushArgs& a) {
  const unsigned long long step = *a.step_ptr;
  const bool lie = a.attack != 0 && a.adv_len > 0 &&
                   ((a.adv_bitmap[step % (unsigned long long)a.adv_len] >> a.worker) & 1u);
  const unsigned long long key = mix64(a.seed ^ (step << 8) ^ (unsigned long long)a.worker);

  // [tile_begin, tile_end): a bucket of the arena.  Buckets are pushed as soon as backprop has finished the layers they
  // cover, on a side stream, so the transfer overlaps the rest of the backward pass (the reference's "send layer l while
  // back-propagating layer l-1", src/model_ops/resnet_split.py:431-623); only the last bucket carries the flag.
  const int tile_end = a.tile_end > 0 ? a.tile_end : a.tv.ntiles;
  for (int tile = a.tile_begin + blockIdx.x; tile < tile_end; tile += gridDim.x) {
    int tensor;
    const int valid = tile_valid(a.tv, tile, tensor);
    const int is_bf16 = a.tv.meta[tensor].is_bf16;
    const long long idx = (long long)tile * DRC_TILE + threadIdx.x * 4;
    const int lane_valid = valid - (int)threadIdx.x * 4;      // elements of this thread that are real
    if constexpr (SIGN) {
      // Thread t holds bits 4(t % 8) .. 4(t % 8) + 3 of word t / 8 of the tile, so the 8 lanes of a lane octet fill one word
      // and a warp's 4 words are 16 contiguous bytes.  Every lane joins the shuffles: padding lanes contribute 0 bits.
      unsigned int bits = 0u;
      if (!(a.src_table && lane_valid <= 0)) {
        const float4 g = push_value<WMOM>(a, lie, key, tensor, is_bf16, idx, lane_valid);
        bits = (unsigned int)(g.x < 0.f) | ((unsigned int)(g.y < 0.f) << 1) | ((unsigned int)(g.z < 0.f) << 2) |
               ((unsigned int)(g.w < 0.f) << 3);
        if (lane_valid < 4) bits &= lane_valid > 0 ? (1u << lane_valid) - 1u : 0u;
      }
      const unsigned int lane = threadIdx.x & 31u;
      unsigned int word = bits << (4u * (lane & 7u));
      word |= __shfl_xor_sync(0xffffffffu, word, 1);
      word |= __shfl_xor_sync(0xffffffffu, word, 2);
      word |= __shfl_xor_sync(0xffffffffu, word, 4);
      const unsigned int w1 = __shfl_sync(0xffffffffu, word, 8), w2 = __shfl_sync(0xffffffffu, word, 16),
                         w3 = __shfl_sync(0xffffffffu, word, 24);
      if (lane == 0) {
        const uint4 q = make_uint4(word, w1, w2, w3);
        const long long widx = (long long)tile * (DRC_TILE / 32) + (threadIdx.x >> 5) * 4;   // this warp's 4 words
        st_f4(reinterpret_cast<float4*>(reinterpret_cast<unsigned int*>(a.dst) + widx), *reinterpret_cast<const float4*>(&q));
        if (a.local_copy) *reinterpret_cast<uint4*>(reinterpret_cast<unsigned int*>(a.local_copy) + widx) = q;
      }
    } else if (WMOM || !a.cyclic) {   // the momentum build has no cyclic path
      if (a.src_table && lane_valid <= 0) continue;             // padding of the slab stays zero, nothing to send
      const float4 g = push_value<WMOM>(a, lie, key, tensor, is_bf16, idx, lane_valid);
      st_f4(reinterpret_cast<float4*>(a.dst + idx), g);
      if (a.local_copy) *reinterpret_cast<float4*>(a.local_copy + idx) = g;
    } else if constexpr (!WMOM) {
      if (a.src_table && lane_valid <= 0) continue;
      float4 re = make_float4(0.f, 0.f, 0.f, 0.f), im = re, plain = re;
#pragma unroll 1
      for (int k = 0; k < a.R; ++k) {
        float4 g = load_grad4(a, k, tensor, is_bf16, idx, lane_valid);
        const float cr = a.coef_re[k], ci = a.coef_im[k];
        re.x = fmaf(cr, g.x, re.x); re.y = fmaf(cr, g.y, re.y); re.z = fmaf(cr, g.z, re.z); re.w = fmaf(cr, g.w, re.w);
        im.x = fmaf(ci, g.x, im.x); im.y = fmaf(ci, g.y, im.y); im.z = fmaf(ci, g.z, im.z); im.w = fmaf(ci, g.w, im.w);
      }
      if (lie) {   // cyclic adversary ADDS to the honest codeword (reference: model_ops/utils.py:8-18)
        float4 e = plain;
        if (a.attack == 1) { e = make_float4(a.magnitude * re.x, a.magnitude * re.y, a.magnitude * re.z, a.magnitude * re.w);
                             im.x += a.magnitude * im.x; im.y += a.magnitude * im.y; im.z += a.magnitude * im.z; im.w += a.magnitude * im.w; }
        else if (a.attack == 2) { e = make_float4(a.magnitude, a.magnitude, a.magnitude, a.magnitude); }
        else if (a.attack == 3) {
          float2 n0 = normal_pair(key, (unsigned long long)idx), n1 = normal_pair(key, (unsigned long long)idx + 2);
          float m = fabsf(a.magnitude);
          e = make_float4(m * n0.x, m * n0.y, m * n1.x, m * n1.y);
        }
        if (lane_valid < 4) {
          if (lane_valid < 1) e.x = 0.f;
          if (lane_valid < 2) e.y = 0.f;
          if (lane_valid < 3) e.z = 0.f;
          e.w = 0.f;
        }
        re.x += e.x; re.y += e.y; re.z += e.z; re.w += e.w;
      }
      float4* d = reinterpret_cast<float4*>(a.dst + 2 * idx);
      st_f4(d, make_float4(re.x, im.x, re.y, im.y));
      st_f4(d + 1, make_float4(re.z, im.z, re.w, im.w));
    }
  }
  return step;
}

__global__ void __launch_bounds__(DRC_THREADS) push_encode_kernel(const __grid_constant__ PushArgs a) {
  const unsigned long long step = push_encode_tiles<false>(a);
  if (grid_last_cta(a.done_counter)) {
    if (threadIdx.x == 0 && a.flag) st_release_sys(a.flag, step);
  }
}

// the momentum build of the non-cyclic push (the cyclic code keeps no worker state)
__global__ void __launch_bounds__(DRC_THREADS) push_encode_wmom_kernel(const __grid_constant__ PushArgs a) {
  const unsigned long long step = push_encode_tiles<true>(a);
  if (grid_last_cta(a.done_counter)) {
    if (threadIdx.x == 0 && a.flag) st_release_sys(a.flag, step);
  }
}

// the signSGD builds (--mode sign_vote): one bit per element, plain and with worker momentum (Signum)
template <bool WMOM>
__global__ void __launch_bounds__(DRC_THREADS) push_encode_sign_kernel(const __grid_constant__ PushArgs a) {
  const unsigned long long step = push_encode_tiles<WMOM, true>(a);
  if (grid_last_cta(a.done_counter)) {
    if (threadIdx.x == 0 && a.flag) st_release_sys(a.flag, step);
  }
}

extern "C" int drc_push_encode(const PushArgs* args, int grid, cudaStream_t stream) {
  if (args->sign) {
    if (args->cyclic) return (int)cudaErrorInvalidValue;
    if (args->wmom) push_encode_sign_kernel<true><<<grid, DRC_THREADS, 0, stream>>>(*args);
    else push_encode_sign_kernel<false><<<grid, DRC_THREADS, 0, stream>>>(*args);
  } else if (args->wmom) {
    if (args->cyclic) return (int)cudaErrorInvalidValue;
    push_encode_wmom_kernel<<<grid, DRC_THREADS, 0, stream>>>(*args);
  } else {
    push_encode_kernel<<<grid, DRC_THREADS, 0, stream>>>(*args);
  }
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Omniscient attack (north-star extension): the Byzantine worker reads the honest workers' slots that
// already landed in PS memory (peer loads over NVLink) and overwrites its own slot with mag * mean(honest).
// ---------------------------------------------------------------------------------------------
struct OmniArgs {
  float* grad_in;                 // peer pointer to the PS arena [P][stride]
  long long slot_stride;          // elements between worker slots
  unsigned int honest_mask;       // workers to average
  int worker;                     // liar's slot
  float magnitude;
  long long total;                // arena elements (multiple of 4)
  unsigned int* done_counter;
  unsigned long long* flag;
  const unsigned long long* step_ptr;
};

__global__ void __launch_bounds__(DRC_THREADS) omniscient_kernel(const __grid_constant__ OmniArgs a) {
  const int nh = __popc(a.honest_mask);
  const float scale = nh > 0 ? a.magnitude / nh : 0.f;
  for (long long i = ((long long)blockIdx.x * DRC_THREADS + threadIdx.x) * 4; i < a.total;
       i += (long long)gridDim.x * DRC_THREADS * 4) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int w = 0; w < DRC_MAX_WORKERS; ++w) {
      if (!((a.honest_mask >> w) & 1u)) continue;
      float4 v = ld_f4(reinterpret_cast<const float4*>(a.grad_in + w * a.slot_stride + i));
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    acc.x *= scale; acc.y *= scale; acc.z *= scale; acc.w *= scale;
    st_f4(reinterpret_cast<float4*>(a.grad_in + a.worker * a.slot_stride + i), acc);
  }
  if (grid_last_cta(a.done_counter)) {
    if (threadIdx.x == 0 && a.flag) st_release_sys(a.flag, *a.step_ptr);
  }
}

extern "C" int drc_omniscient(const OmniArgs* args, int grid, cudaStream_t stream) {
  omniscient_kernel<<<grid, DRC_THREADS, 0, stream>>>(*args);
  return (int)cudaGetLastError();
}

extern "C" int drc_sizeof_PushArgs() { return (int)sizeof(PushArgs); }
extern "C" int drc_sizeof_OmniArgs() { return (int)sizeof(OmniArgs); }
