// Memory-bound kernels: SGD step, FedAvg on flat arenas, fused loss fwd+bwd, eval, argmax,
// min-max scaling, keyed permutation, dtype conversion.  All are single-pass, 128-bit vectorised
// where alignment allows, and sized as a persistent grid (132 SMs of an H100 SXM x 8 CTAs) with grid-stride loops.
//
// Parity map (SURVEY §2.5b): K9 sigmoid+BCE (client_federated.py:65,79), K10 softmax-xent (BASELINE
// 2-logit configs), K11 SSE (cf.py:112,158), K12 SGD (fc.py:355; cf.py:206-207), K13 MinMax
// (datasets.py:31-32), K14 shuffled sampling (cf.py:203), K15 eval (cf.py:233-253), K16 argmax
// (fc.py:252-256), K3 FedAvg (fc.py:373,568).
#include "colearn_kernels.h"

#include <cuda_bf16.h>
#include <math.h>

namespace colearn {
namespace {

constexpr int kThreads = 256;
inline int grid_for(int64_t n, int per_thread = 4) {
  int64_t b = (n + (int64_t)kThreads * per_thread - 1) / ((int64_t)kThreads * per_thread);
  const int64_t cap = 132 * 8;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float block_sum(float v, float* scratch /*[32]*/) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) scratch[w] = v;
  __syncthreads();
  if (w == 0) {
    v = lane < (blockDim.x >> 5) ? scratch[lane] : 0.f;
    v = warp_sum(v);
  }
  __syncthreads();
  return v;  // valid in warp 0
}

// ---- SGD ---------------------------------------------------------------------------------------
__global__ void sgd_step_kernel(float* __restrict__ p, const float* __restrict__ g, float lr, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool aligned = ((((uintptr_t)p) | ((uintptr_t)g)) & 15) == 0;
  if (aligned) {
    const int64_t n4 = n >> 2;
    float4* p4 = reinterpret_cast<float4*>(p);
    const float4* g4 = reinterpret_cast<const float4*>(g);
    for (int64_t j = i; j < n4; j += stride) {
      float4 a = p4[j];
      const float4 b = __ldg(g4 + j);
      a.x = fmaf(-lr, b.x, a.x); a.y = fmaf(-lr, b.y, a.y);
      a.z = fmaf(-lr, b.z, a.z); a.w = fmaf(-lr, b.w, a.w);
      p4[j] = a;
    }
    for (int64_t j = (n4 << 2) + i; j < n; j += stride) p[j] = fmaf(-lr, g[j], p[j]);
  } else {
    for (; i < n; i += stride) p[i] = fmaf(-lr, g[i], p[i]);
  }
}

// p *= scale in place: a rank pre-scales its trained arena by its FedAvg weight n_k / sum n (0 for a rank that was not
// selected) so that the in-switch multimem.ld_reduce of the two-shot kernel — which sums every member of the multicast group
// with equal weight — yields the weighted / subset average (SURVEY 7.3-4)
__global__ void scale_inplace_kernel(float* __restrict__ p, float scale, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if ((((uintptr_t)p) & 15) == 0) {
    const int64_t n4 = n >> 2;
    float4* p4 = reinterpret_cast<float4*>(p);
    for (int64_t j = i; j < n4; j += stride) {
      float4 a = p4[j];
      a.x *= scale; a.y *= scale; a.z *= scale; a.w *= scale;
      p4[j] = a;
    }
    for (int64_t j = (n4 << 2) + i; j < n; j += stride) p[j] *= scale;
  } else {
    for (int64_t j = i; j < n; j += stride) p[j] *= scale;
  }
}

__global__ void sgd_step_bf16grad_kernel(float* __restrict__ p, const __nv_bfloat16* __restrict__ g,
                                         float lr, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    p[i] = fmaf(-lr, __bfloat162float(g[i]), p[i]);
}

// ---- FedAvg on flat arenas ------------------------------------------------------------------------
template <bool APPLY>
__global__ void fedavg_kernel(float* __restrict__ theta, const float* __restrict__ slots,
                              int64_t slot_stride, const float* __restrict__ weights, int k,
                              float server_lr, int64_t n) {
  // no cap on the number of workers (the coordinator's upper bound is 100, selection 'all' applies none): the first
  // kSw weights are staged in shared memory, any beyond that are read through the read-only cache
  constexpr int kSw = 256;
  __shared__ float sw[kSw];
  for (int c = threadIdx.x; c < k && c < kSw; c += blockDim.x) sw[c] = weights[c];
  __syncthreads();
  auto wt = [&](int c) -> float { return c < kSw ? sw[c] : __ldg(weights + c); };
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool aligned = (((uintptr_t)theta | (uintptr_t)slots) & 15) == 0 && (slot_stride & 3) == 0;
  if (aligned) {
    const int64_t n4 = n >> 2;
    for (int64_t j = i0; j < n4; j += stride) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int c = 0; c < k; ++c) {
        const float4 v = __ldcs(reinterpret_cast<const float4*>(slots + c * slot_stride) + j);
        const float w = wt(c);
        acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y);
        acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
      }
      float4* t4 = reinterpret_cast<float4*>(theta) + j;
      if (APPLY) {
        float4 t = *t4;
        t.x = fmaf(server_lr, acc.x - t.x, t.x); t.y = fmaf(server_lr, acc.y - t.y, t.y);
        t.z = fmaf(server_lr, acc.z - t.z, t.z); t.w = fmaf(server_lr, acc.w - t.w, t.w);
        *t4 = t;
      } else {
        *t4 = acc;
      }
    }
    for (int64_t j = (n4 << 2) + i0; j < n; j += stride) {
      float acc = 0.f;
      for (int c = 0; c < k; ++c) acc = fmaf(wt(c), slots[c * slot_stride + j], acc);
      theta[j] = APPLY ? fmaf(server_lr, acc - theta[j], theta[j]) : acc;
    }
  } else {
    for (int64_t j = i0; j < n; j += stride) {
      float acc = 0.f;
      for (int c = 0; c < k; ++c) acc = fmaf(wt(c), slots[c * slot_stride + j], acc);
      theta[j] = APPLY ? fmaf(server_lr, acc - theta[j], theta[j]) : acc;
    }
  }
}

// FedAvg average (same weights, same summation order as fedavg_kernel) followed by a server optimizer step (server_opt.cuh)
// on theta with the moments opt.m[n] / opt.v[n]: Coordinator-side FedAvgM / FedAdagrad / FedAdam / FedYogi in one pass
__global__ void fedavg_opt_kernel(float* __restrict__ theta, const float* __restrict__ slots, int64_t slot_stride,
                                  const float* __restrict__ weights, int k, ServerOptArgs opt, int64_t n) {
  constexpr int kSw = 256;
  __shared__ float sw[kSw];
  for (int c = threadIdx.x; c < k && c < kSw; c += blockDim.x) sw[c] = weights[c];
  __syncthreads();
  auto wt = [&](int c) -> float { return c < kSw ? sw[c] : __ldg(weights + c); };
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool aligned = (((uintptr_t)theta | (uintptr_t)slots | (uintptr_t)opt.m | (uintptr_t)opt.v) & 15) == 0 && (slot_stride & 3) == 0;
  int64_t scalar_from = 0;
  if (aligned) {
    const int64_t n4 = n >> 2;
    for (int64_t j = i0; j < n4; j += stride) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int c = 0; c < k; ++c) {
        const float4 v = __ldcs(reinterpret_cast<const float4*>(slots + c * slot_stride) + j);
        const float w = wt(c);
        acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y);
        acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
      }
      float4* t4 = reinterpret_cast<float4*>(theta) + j;
      *t4 = server_opt_step4(opt, j, *t4, acc);
    }
    scalar_from = n4 << 2;
  }
  for (int64_t j = scalar_from + i0; j < n; j += stride) {
    float acc = 0.f;
    for (int c = 0; c < k; ++c) acc = fmaf(wt(c), slots[c * slot_stride + j], acc);
    theta[j] = server_opt_step(opt, j, theta[j], acc);
  }
}

// Slot loaders of the robust FedAvg body.  stream(c, j) / cached(c, j): value j of slot c, read once (register path) or
// reread through L1 / L2 (general path); average(a, t): the a the server step moves towards, from the aggregate of the slots.
// fp32 slots hold the client models themselves.
struct F32Slots {
  const float* p;
  int64_t stride;
  __device__ __forceinline__ float stream(int c, int64_t j) const { return __ldcs(p + c * stride + j); }
  __device__ __forceinline__ float cached(int c, int64_t j) const { return __ldg(p + c * stride + j); }
  __device__ __forceinline__ float average(float a, float) const { return a; }
};
// Quantized slots (uplink_quant.cuh) hold the clients' deltas: value j is decoded from its code and its block's step (one
// broadcast load per warp: the 32 elements of a warp lie in one block), and a = theta + aggregate of the decoded deltas
// (theta + x is monotone in x: the robust aggregate of the decoded models up to the final add).
template <int BITS>
struct QSlots {
  const uint8_t* payload;
  int64_t row_bytes;
  const float* scales;
  int64_t nblk;
  __device__ __forceinline__ float cached(int c, int64_t j) const {
    const float step = __ldg(scales + c * nblk + (j >> 8));
    int q;
    if constexpr (BITS == 8) {
      q = (int)(int8_t)__ldg(payload + c * row_bytes + j);
    } else {
      q = uq_nibble(__ldg(payload + c * row_bytes + (j >> 1)), (int)(j & 1));
    }
    return uq_decode(q, step);
  }
  __device__ __forceinline__ float stream(int c, int64_t j) const { return cached(c, j); }
  __device__ __forceinline__ float average(float a, float t) const { return t + a; }
};

// Byzantine-robust aggregate (robust_agg.cuh: coordinate-wise median / trimmed mean over all k slots, unweighted) followed by
// theta += opt.lr (a - theta) (opt.kind 0) or a server optimizer step (server_opt.cuh).  One element per thread.
// KMAX > 0: register path for k <= KMAX, the k values and their keys stay in registers and the rank count is KMAX x KMAX
// unrolled compares; KMAX = 0: any k, tiles of 32 values in registers, the rank count rereads the values through L1 / L2
// (k ceil(k / 32) loads per element).
template <int KMAX, class Slots>
__device__ __forceinline__ void fedavg_robust_body(float* __restrict__ theta, const Slots& slots, int k, const AggArgs& agg,
                                                   const ServerOptArgs& opt, int64_t n) {
  const int b = agg_trim_count(agg, k);
  const uint32_t valid = k >= 32 ? 0xffffffffu : (1u << k) - 1u;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    float a;
    if constexpr (KMAX > 0) {
      float v[KMAX];
#pragma unroll
      for (int c = 0; c < KMAX; ++c) v[c] = c < k ? slots.stream(c, j) : 0.f;
      a = agg_robust<KMAX>(v, valid, k, b);
    } else {
      a = agg_robust_tiled<32>([&](int c) { return slots.cached(c, j); }, k, b);
    }
    const float t = theta[j];
    a = slots.average(a, t);
    theta[j] = (opt.kind == SOPT_SGD) ? fmaf(opt.lr, a - t, t) : server_opt_step(opt, j, t, a);
  }
}

template <int KMAX>
__global__ void __launch_bounds__(256)
fedavg_robust_kernel(float* __restrict__ theta, const float* __restrict__ slots, int64_t slot_stride, int k, AggArgs agg,
                     ServerOptArgs opt, int64_t n) {
  fedavg_robust_body<KMAX>(theta, F32Slots{slots, slot_stride}, k, agg, opt, n);
}

// ---- codec kernels: the per-lane steps they share ------------------------------------------------------------------------------
// Every codec kernel below runs one warp per 256-element block (kUqBlock) and lane l holds elements e0 .. e0 + 7 of its block,
// e0 = 256 b + 8 l.  Each kernel decides its own `vec` (its pointers 16-byte aligned, and whatever else it needs); without it
// the same bits move through scalar accesses.

// the cache hint of a load: plain (data the kernel writes back), streaming __ldcs (read once) or read-only __ldg
enum LdHint { kLdPlain, kLdStream, kLdReadOnly };
template <LdHint HINT, class T>
__device__ __forceinline__ T ld_hint(const T* p) {
  if constexpr (HINT == kLdStream) return __ldcs(p);
  else if constexpr (HINT == kLdReadOnly) return __ldg(p);
  else return *p;
}

// lane l's elements e0 .. e0 + 7 of p, 0 past n: two 16-byte loads with hint HINT when vec, which must imply n % 4 == 0 (a
// 4-element group is then wholly inside or past n), plain scalar loads otherwise.  One branch on vec and predicated loads
// inside it: a branch per group between a 16-byte and scalar loads kept a lane's loads from overlapping (the encoders ran up
// to a quarter slower on the H100).
template <LdHint HINT>
__device__ __forceinline__ void lane_load8(const float* __restrict__ p, int64_t e0, int64_t n, bool vec, float (&x)[8]) {
  if (vec) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (e0 + 4 * h < n) v = ld_hint<HINT>(reinterpret_cast<const float4*>(p + e0 + 4 * h));
      x[4 * h + 0] = v.x; x[4 * h + 1] = v.y; x[4 * h + 2] = v.z; x[4 * h + 3] = v.w;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = e0 + i < n ? p[e0 + i] : 0.f;
  }
}

// lane l's elements e0 .. e0 + 7 of p back, none past n: 16-byte stores of the groups of 4 inside n when vec, scalar stores
// otherwise (any n)
__device__ __forceinline__ void lane_store8(float* __restrict__ p, int64_t e0, int64_t n, bool vec, const float (&x)[8]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t e = e0 + 4 * h;
    if (vec && e + 4 <= n) {
      *reinterpret_cast<float4*>(p + e) = make_float4(x[4 * h], x[4 * h + 1], x[4 * h + 2], x[4 * h + 3]);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (e + i < n) p[e + i] = x[4 * h + i];
      }
    }
  }
}

// the block's step and inverse scale (uq_block_scale) from the lanes' deltas d: the warp max of uq_abs_bits by shuffles
template <int BITS>
__device__ __forceinline__ void warp_block_scale(const float (&d)[8], float& step, float& inv) {
  uint32_t amax = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint32_t a = uq_abs_bits(d[i]);
    amax = a > amax ? a : amax;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const uint32_t a = __shfl_xor_sync(0xffffffffu, amax, o);
    amax = a > amax ? a : amax;
  }
  uq_block_scale(amax, UqCodec<BITS>::kLevels, step, inv);
}

// lane l's 8 codes into / out of a payload row: one 8-byte (int8) or 4-byte (int4, element 2 i in the low nibble) access
template <int BITS>
__device__ __forceinline__ void store_codes8(uint8_t* __restrict__ row, int64_t e0, const int (&q)[8]) {
  if constexpr (BITS == 8) {
    uint2 w = make_uint2(0u, 0u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      w.x |= ((uint32_t)q[i] & 0xffu) << (8 * i);
      w.y |= ((uint32_t)q[4 + i] & 0xffu) << (8 * i);
    }
    *reinterpret_cast<uint2*>(row + e0) = w;
  } else {
    uint32_t w = 0u;
#pragma unroll
    for (int i = 0; i < 8; ++i) w |= ((uint32_t)q[i] & 0xfu) << (4 * i);
    *reinterpret_cast<uint32_t*>(row + (e0 >> 1)) = w;
  }
}
template <int BITS, LdHint HINT>
__device__ __forceinline__ void load_codes8(const uint8_t* __restrict__ row, int64_t e0, int (&q)[8]) {
  if constexpr (BITS == 8) {
    const uint2 w = ld_hint<HINT>(reinterpret_cast<const uint2*>(row + e0));
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      q[i] = (int)(int8_t)(w.x >> (8 * i));
      q[4 + i] = (int)(int8_t)(w.y >> (8 * i));
    }
  } else {
    const uint32_t w = ld_hint<HINT>(reinterpret_cast<const unsigned int*>(row + (e0 >> 1)));
#pragma unroll
    for (int i = 0; i < 8; ++i) q[i] = uq_nibble(w, i);
  }
}

// The FedAvg weights of the codec apply kernels, as in fedavg_kernel: the first kSw staged in the shared array sw by the whole
// CTA (the constructor ends in __syncthreads), any beyond read through the read-only cache.
struct StagedWeights {
  static constexpr int kSw = 256;
  const float* sw;
  const float* weights;
  __device__ __forceinline__ StagedWeights(float* s, const float* w, int k) : sw(s), weights(w) {
    for (int c = threadIdx.x; c < k && c < kSw; c += blockDim.x) s[c] = w[c];
    __syncthreads();
  }
  __device__ __forceinline__ float wt(int c) const { return c < kSw ? sw[c] : __ldg(weights + c); }
};

// theta[e0 .. e0 + 7] (none past n) moved towards a = theta + acc: theta += opt.lr (a - theta) (OPT false) or the server
// optimizer step (OPT true); 16-byte accesses of theta and the moments per 4 elements inside n when vec
template <bool OPT>
__device__ __forceinline__ void apply8(float* __restrict__ theta, int64_t e0, int64_t n, bool vec, const float (&acc)[8],
                                       const ServerOptArgs& opt) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t e = e0 + 4 * h;
    if (vec && e + 4 <= n) {
      float4* t4 = reinterpret_cast<float4*>(theta + e);
      float4 t = *t4;
      const float4 a = make_float4(t.x + acc[4 * h], t.y + acc[4 * h + 1], t.z + acc[4 * h + 2], t.w + acc[4 * h + 3]);
      if constexpr (OPT) {
        t = server_opt_step4(opt, e >> 2, t, a);
      } else {
        t.x = fmaf(opt.lr, a.x - t.x, t.x); t.y = fmaf(opt.lr, a.y - t.y, t.y);
        t.z = fmaf(opt.lr, a.z - t.z, t.z); t.w = fmaf(opt.lr, a.w - t.w, t.w);
      }
      *t4 = t;
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (e + i < n) {
          const float t = theta[e + i], a = t + acc[4 * h + i];
          theta[e + i] = OPT ? server_opt_step(opt, e + i, t, a) : fmaf(opt.lr, a - t, t);
        }
      }
    }
  }
}

// ---- uplink codec (uplink_quant.cuh) ----------------------------------------------------------------------------------------
// Encode: one warp per (row, block).  The lanes load the model (streamed) and theta, the warp takes the block's step, every
// lane stores its 8 codes and lane 0 the step.  Elements past n encode as 0 (the int4 pad nibble).  Single pass.
template <int BITS>
__global__ void __launch_bounds__(256)
quantize_delta_kernel(const float* __restrict__ models, int64_t model_stride, const float* __restrict__ theta,
                      const uint32_t* __restrict__ keys, int k, uint8_t* __restrict__ payload, int64_t row_bytes,
                      float* __restrict__ scales, int64_t n) {
  const int lane = threadIdx.x & 31;
  const int64_t nblk = uq_nblk(n);
  const int64_t tasks = nblk * k;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const bool vec = (((uintptr_t)models | (uintptr_t)theta) & 15) == 0 && (model_stride & 3) == 0 && (n & 3) == 0;
  for (int64_t t = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < tasks; t += warps) {
    const int c = (int)(t / nblk);
    const int64_t blk = t - (int64_t)c * nblk;
    const int64_t e0 = blk * kUqBlock + lane * 8;
    float m[8], th[8], d[8];
    lane_load8<kLdStream>(models + c * model_stride, e0, n, vec, m);
    lane_load8<kLdReadOnly>(theta, e0, n, vec, th);
#pragma unroll
    for (int i = 0; i < 8; ++i) d[i] = m[i] - th[i];
    float step, inv;
    warp_block_scale<BITS>(d, step, inv);
    const uint32_t key = keys[c];
    if (e0 < n) {
      int q[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) q[i] = uq_encode(d[i], inv, key, (uint32_t)(e0 + i), UqCodec<BITS>::kLevels);
      store_codes8<BITS>(payload + c * row_bytes, e0, q);
    }
    if (lane == 0) scales[c * nblk + blk] = step;
  }
}

// Decode + FedAvg reduce + apply, the quantized twin of fedavg_kernel / fedavg_opt_kernel: per element
// acc = fmaf(w_k, d^_k, acc) in slot order from +0, a = theta + acc, then theta += opt.lr (a - theta) (OPT false) or the server
// optimizer step (OPT true).  One warp per block: a slot's step is one broadcast load per warp, its codes one streamed load per
// lane.
template <int BITS, bool OPT>
__global__ void __launch_bounds__(256)
fedavg_q_kernel(float* __restrict__ theta, const uint8_t* __restrict__ payload, int64_t row_bytes, const float* __restrict__ scales,
                const float* __restrict__ weights, int k, ServerOptArgs opt, int64_t n) {
  __shared__ float sw[StagedWeights::kSw];
  const StagedWeights staged(sw, weights, k);
  const int lane = threadIdx.x & 31;
  const int64_t nblk = uq_nblk(n);
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const bool vec = (((uintptr_t)theta | (uintptr_t)opt.m | (uintptr_t)opt.v) & 15) == 0;
  for (int64_t blk = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); blk < nblk; blk += warps) {
    const int64_t e0 = blk * kUqBlock + lane * 8;
    if (e0 >= n) continue;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll 4
    for (int c = 0; c < k; ++c) {
      const float step = __ldg(scales + c * nblk + blk);
      const float w = staged.wt(c);
      int q[8];
      load_codes8<BITS, kLdStream>(payload + c * row_bytes, e0, q);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(w, uq_decode(q[i], step), acc[i]);
    }
    apply8<OPT>(theta, e0, n, vec, acc, opt);
  }
}

// robust aggregate of the decoded deltas: the body of fedavg_robust_kernel with the decoding loader
template <int KMAX, int BITS>
__global__ void __launch_bounds__(256)
fedavg_q_robust_kernel(float* __restrict__ theta, const uint8_t* __restrict__ payload, int64_t row_bytes, const float* __restrict__ scales,
                       int k, AggArgs agg, ServerOptArgs opt, int64_t n) {
  fedavg_robust_body<KMAX>(theta, QSlots<BITS>{payload, row_bytes, scales, uq_nblk(n)}, k, agg, opt, n);
}

// ---- distance-based robust aggregation (distance_agg.cuh) ---------------------------------------------------------------------
// Every pass walks the fixed 2048-element chunks grid-stride, one chunk per CTA at a time, lane t holding elements
// 2048 q + 8 t .. + 7 (the codec kernels' warp-per-256-block layout).  Row loaders: load8<HINT>(k, e0, x) = elements e0 .. e0 + 7
// of row k, 0 past n (e0 < n); kDelta: the rows are deltas (c^0 = 0, theta added at the end) rather than models (c^0 = theta).
struct F32Rows {
  static constexpr bool kDelta = false;
  const float* p;
  int64_t stride, n;
  bool vec;
  template <LdHint HINT>
  __device__ __forceinline__ void load8(int k, int64_t e0, float (&x)[8]) const { lane_load8<HINT>(p + k * stride, e0, n, vec, x); }
};
template <int BITS>
struct QRows {
  static constexpr bool kDelta = true;
  const uint8_t* payload;
  int64_t row_bytes;
  const float* scales;
  int64_t nblk, n;
  template <LdHint HINT>
  __device__ __forceinline__ void load8(int k, int64_t e0, float (&x)[8]) const {
    const float step = __ldg(scales + k * nblk + (e0 >> 8));
    int q[8];
    load_codes8<BITS, HINT>(payload + k * row_bytes, e0, q);
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = e0 + i < n ? uq_decode(q[i], step) : 0.f;   // codes past n are padding
  }
};

__device__ __forceinline__ double warp_tree_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The per-row chunk sums of one CTA: put(r, s) adds row r's lane values over the warp into red[warp][r % 32]; flush writes rows
// r0 .. r0 + rows - 1 (rows <= 32) as the warp sums added in warp order.  Every thread of the CTA calls both.
struct DaRowSums {
  double (*red)[32];
  __device__ __forceinline__ void put(int r, double s) const {
    s = warp_tree_f64(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][r & 31] = s;
  }
  __device__ __forceinline__ void flush(int r0, int rows, double* __restrict__ partial, int64_t nchunks, int64_t q) const {
    __syncthreads();
    if ((int)threadIdx.x < rows) {
      double t = red[0][threadIdx.x];
#pragma unroll
      for (int w = 1; w < kDaThreads / 32; ++w) t += red[w][threadIdx.x];
      partial[(int64_t)(r0 + threadIdx.x) * nchunks + q] = t;
    }
    __syncthreads();
  }
};

// lane's start point c^0: theta (models) or 0 (deltas)
template <class Rows>
__device__ __forceinline__ void da_start8(const float* __restrict__ theta, int64_t e0, int64_t n, bool vec, float (&c)[8]) {
  if constexpr (Rows::kDelta) {
#pragma unroll
    for (int i = 0; i < 8; ++i) c[i] = 0.f;
  } else {
    lane_load8<kLdReadOnly>(theta, e0, n, vec, c);
  }
}

// Distance pass of the first step: the chunk sums of (x_k - c^0)^2 for every row
template <class Rows>
__global__ void __launch_bounds__(kDaThreads)
dagg_dist_kernel(Rows rows, const float* __restrict__ theta, int k, DistAggScratch sc, int64_t n) {
  __shared__ double red[kDaThreads / 32][32];
  const DaRowSums sums{red};
  const int64_t nchunks = da_chunks(n);
  const bool vec = ((uintptr_t)theta & 15) == 0 && (n & 3) == 0;
  for (int64_t q = blockIdx.x; q < nchunks; q += gridDim.x) {
    const int64_t e0 = q * kDaChunk + threadIdx.x * 8;
    float c[8];
    da_start8<Rows>(theta, e0, n, vec, c);
    for (int r0 = 0; r0 < k; r0 += 32) {
      const int nr = k - r0 < 32 ? k - r0 : 32;
      for (int r = 0; r < nr; ++r) {
        float x[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (e0 < n) rows.template load8<kLdStream>(r0 + r, e0, x);
        sums.put(r, da_lane_sq8(x, c));
      }
      sums.flush(r0, nr, sc.partial, nchunks, q);
    }
  }
}

// A geomed step l < L fused with the next distance pass: the lane forms c^l for its 8 elements from the current weights (c^0
// when no row is left), then the chunk sums of (x_k - c^l)^2, in one read of the rows.  KMAX > 0: k <= KMAX, the rows' 8 values
// stay in registers between the two loops; KMAX = 0: any k, the second loop rereads them through L1 / L2.
template <int KMAX, class Rows>
__global__ void __launch_bounds__(kDaThreads, 1)
dagg_center_kernel(Rows rows, const float* __restrict__ theta, int k, DistAggScratch sc, int64_t n) {
  __shared__ double red[kDaThreads / 32][32];
  __shared__ float sw[StagedWeights::kSw];
  const StagedWeights staged(sw, sc.w, k);
  const DaRowSums sums{red};
  const bool live = *sc.live > 0;
  const int64_t nchunks = da_chunks(n);
  const bool vec = ((uintptr_t)theta & 15) == 0 && (n & 3) == 0;
  for (int64_t q = blockIdx.x; q < nchunks; q += gridDim.x) {
    const int64_t e0 = q * kDaChunk + threadIdx.x * 8;
    const bool in = e0 < n;
    float c[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if constexpr (KMAX > 0) {
      float x[KMAX][8];
#pragma unroll
      for (int r = 0; r < KMAX; ++r) {
        float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (r < k && in) rows.template load8<kLdStream>(r, e0, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) x[r][i] = v[i];
      }
#pragma unroll
      for (int r = 0; r < KMAX; ++r) {
        const float w = r < k ? staged.wt(r) : 0.f;
        if (w != 0.f) {
#pragma unroll
          for (int i = 0; i < 8; ++i) c[i] = fmaf(w, x[r][i], c[i]);
        }
      }
      if (!live) da_start8<Rows>(theta, e0, n, vec, c);
#pragma unroll
      for (int r = 0; r < KMAX; ++r) {
        if (r < k) sums.put(r, da_lane_sq8(x[r], c));
      }
      sums.flush(0, k, sc.partial, nchunks, q);
    } else {
      if (in) {
        for (int r = 0; r < k; ++r) {
          const float w = staged.wt(r);
          if (w != 0.f) {
            float x[8];
            rows.template load8<kLdReadOnly>(r, e0, x);
#pragma unroll
            for (int i = 0; i < 8; ++i) c[i] = fmaf(w, x[i], c[i]);
          }
        }
      }
      if (!live) da_start8<Rows>(theta, e0, n, vec, c);
      for (int r0 = 0; r0 < k; r0 += 32) {
        const int nr = k - r0 < 32 ? k - r0 : 32;
        for (int r = 0; r < nr; ++r) {
          float x[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          if (in) rows.template load8<kLdReadOnly>(r0 + r, e0, x);
          sums.put(r, da_lane_sq8(x, c));
        }
        sums.flush(r0, nr, sc.partial, nchunks, q);
      }
    }
  }
}

// Finalisation of one step: CTA r adds row r's chunk sums (distance_agg.cuh order) into d_r; the last CTA to take a ticket
// forms the raw weights in parallel, their sum in row order (thread 0) and the weights, and leaves the ticket at 0.
__global__ void __launch_bounds__(kDaThreads)
dagg_finalize_kernel(DistAggScratch sc, const float* __restrict__ alpha, int k, DistAggArgs g, float* __restrict__ w_out, int64_t nchunks) {
  __shared__ double red[kDaThreads / 32];
  __shared__ double s_tot;
  __shared__ int s_last;
  const int r = blockIdx.x;
  double v = 0.0;
  for (int64_t q = threadIdx.x; q < nchunks; q += kDaThreads) v += __ldcg(sc.partial + (int64_t)r * nchunks + q);
  v = warp_tree_f64(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = red[0];
#pragma unroll
    for (int w = 1; w < kDaThreads / 32; ++w) t += red[w];
    sc.dist[r] = sqrt(t);
    __threadfence();                    // d_r visible device-wide before the ticket
    s_last = atomicAdd(sc.ticket, 1u) == (unsigned)(k - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int i = threadIdx.x; i < k; i += kDaThreads) sc.raw[i] = da_raw(g, alpha[i], __ldcg(sc.dist + i));
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    int live = 0;
    for (int i = 0; i < k; ++i) {
      tot += sc.raw[i];
      live += da_kept(__ldcg(sc.dist + i)) ? 1 : 0;
    }
    if (!(tot > 0.0)) live = 0;
    s_tot = tot;
    *sc.live = live;
    *sc.ticket = 0u;
    s_last = live;
  }
  __syncthreads();
  const double tot = s_tot;
  const bool any = s_last > 0;
  for (int i = threadIdx.x; i < k; i += kDaThreads) {
    const float w = any ? da_weight(g, sc.raw[i], __ldcg(sc.dist + i), tot) : 0.f;
    sc.w[i] = w;
    if (w_out != nullptr) w_out[i] = w;
  }
}

// theta[e0 .. e0 + 7] (t, none past n) moved towards a: theta += opt.lr (a - theta) (OPT false) or the server optimizer step
// (OPT true); 16-byte accesses of theta and the moments per 4 elements inside n when vec
template <bool OPT>
__device__ __forceinline__ void step_to8(float* __restrict__ theta, int64_t e0, int64_t n, bool vec, const float (&t)[8],
                                         const float (&a)[8], const ServerOptArgs& opt) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t e = e0 + 4 * h;
    if (vec && e + 4 <= n) {
      float4 tt = make_float4(t[4 * h], t[4 * h + 1], t[4 * h + 2], t[4 * h + 3]);
      const float4 aa = make_float4(a[4 * h], a[4 * h + 1], a[4 * h + 2], a[4 * h + 3]);
      if constexpr (OPT) {
        tt = server_opt_step4(opt, e >> 2, tt, aa);
      } else {
        tt.x = fmaf(opt.lr, aa.x - tt.x, tt.x); tt.y = fmaf(opt.lr, aa.y - tt.y, tt.y);
        tt.z = fmaf(opt.lr, aa.z - tt.z, tt.z); tt.w = fmaf(opt.lr, aa.w - tt.w, tt.w);
      }
      *reinterpret_cast<float4*>(theta + e) = tt;
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (e + i < n) {
          const float tv = t[4 * h + i], av = a[4 * h + i];
          theta[e + i] = OPT ? server_opt_step(opt, e + i, tv, av) : fmaf(opt.lr, av - tv, tv);
        }
      }
    }
  }
}

// Last pass: the aggregate from the final weights (geomed: c^L, or c^0 when no row is left; norm_clip: c^0 + the clipped sum),
// theta + it for deltas, and the server step on theta with the moments in place.
template <class Rows, bool CLIP, bool OPT>
__global__ void __launch_bounds__(kDaThreads)
dagg_apply_kernel(Rows rows, float* __restrict__ theta, int k, DistAggScratch sc, ServerOptArgs opt, int64_t n) {
  __shared__ float sw[StagedWeights::kSw];
  const StagedWeights staged(sw, sc.w, k);
  const bool live = *sc.live > 0;
  const int64_t nchunks = da_chunks(n);
  const bool vec = (((uintptr_t)theta | (uintptr_t)opt.m | (uintptr_t)opt.v) & 15) == 0 && (n & 3) == 0;
  for (int64_t q = blockIdx.x; q < nchunks; q += gridDim.x) {
    const int64_t e0 = q * kDaChunk + threadIdx.x * 8;
    if (e0 >= n) continue;
    float t[8], c0[8], acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    lane_load8<kLdPlain>(theta, e0, n, vec, t);
#pragma unroll
    for (int i = 0; i < 8; ++i) c0[i] = Rows::kDelta ? 0.f : t[i];
#pragma unroll 4
    for (int r = 0; r < k; ++r) {
      const float w = staged.wt(r);
      if (w != 0.f) {
        float x[8];
        rows.template load8<kLdStream>(r, e0, x);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(w, CLIP ? x[i] - c0[i] : x[i], acc[i]);
      }
    }
    float a[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      a[i] = CLIP ? c0[i] + acc[i] : (live ? acc[i] : c0[i]);
      if (Rows::kDelta) a[i] = t[i] + a[i];
    }
    step_to8<OPT>(theta, e0, n, vec, t, a, opt);
  }
}

// ---- top-k uplink with error feedback (uplink_topk.cuh) -----------------------------------------------------------------------
// exclusive prefix over the lower lanes of x in [0, 15], one ballot per bit
__device__ __forceinline__ int warp_exclusive_prefix4(int x, uint32_t lower_lanes) {
  int s = 0;
#pragma unroll
  for (int b = 0; b < 4; ++b) s += __popc(__ballot_sync(0xffffffffu, (x >> b) & 1) & lower_lanes) << b;
  return s;
}

// The selection of one 256-element block by its warp, lane l holding the keys of elements 8 l .. 8 l + 7: the warp finds the
// k_b-th greatest key T bit by bit from the top (31 rounds of one __reduce_add_sync: the largest T with #{key >= T} >= k_b),
// keeps every key > T and the lowest-index keys == T up to k_b (a ballot prefix of the per-lane tie counts).  keep[i] flags
// this lane's kept elements, `first` is the lane's first entry in the block (the exclusive prefix of the per-lane kept
// counts), so that the kept entries land in index order.  Keys in and flags out by value: passed by reference, the routine
// changed the register allocation of topk_delta_kernel.
struct TopkKeys8 { uint32_t key[8]; };
struct TopkSel8 { bool keep[8]; int first; };
__device__ __forceinline__ TopkSel8 warp_topk_select(TopkKeys8 keys, int kb, uint32_t lower_lanes) {
  const uint32_t* key = keys.key;
  TopkSel8 sel;
  uint32_t thr = 0;
  for (int b = 30; b >= 0; --b) {                   // keys are below 2^31
    const uint32_t cand = thr | (1u << b);
    int cnt = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) cnt += key[i] >= cand ? 1 : 0;
    if (__reduce_add_sync(0xffffffffu, cnt) >= kb) thr = cand;
  }
  int ngt = 0, ntie = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    ngt += key[i] > thr ? 1 : 0;
    ntie += key[i] == thr ? 1 : 0;
  }
  // ties this lane may keep: the kb - #{key > thr} >= 1 lowest-index ties of the block, minus those of the lower lanes
  const int room = kb - __reduce_add_sync(0xffffffffu, ngt) - warp_exclusive_prefix4(ntie, lower_lanes);
  // per-element flags, not a bit mask: a `keep |= 1u << i` form of this selection lost element 1's tie on the H100
  // (sm_90a, CUDA 12.9) while its PTX and the SIMT build were right
  int nkeep = 0, seen = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const bool tie = key[i] == thr;
    sel.keep[i] = key[i] > thr || (tie && seen < room);
    seen += tie ? 1 : 0;
    nkeep += sel.keep[i] ? 1 : 0;
  }
  sel.first = warp_exclusive_prefix4(nkeep, lower_lanes);
  return sel;
}

// a lane's kept entries (offset in the block, value v[i]) in index order from entry `out` + sel.first of the wire
__device__ __forceinline__ void topk_emit(uint8_t* __restrict__ indices, float* __restrict__ values, int64_t out, int lane,
                                          const TopkSel8& sel, const float (&v)[8]) {
  int o = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (sel.keep[i]) {
      indices[out + sel.first + o] = (uint8_t)(lane * 8 + i);
      values[out + sel.first + o] = v[i];
      ++o;
    }
  }
}

// Encode: one warp per (row, block).  The lanes load the model (streamed), theta and the residual, warp_topk_select picks the
// entries, and the residual is written back in place.  Elements past n take key 0: they lose every tie to the block's own
// elements, and k_b <= m_b.
__global__ void __launch_bounds__(256)
topk_delta_kernel(const float* __restrict__ models, int64_t model_stride, const float* __restrict__ theta, float* __restrict__ residual,
                  int64_t residual_stride, int k, int topk, uint8_t* __restrict__ indices, float* __restrict__ values, int64_t entries,
                  int64_t n) {
  const int lane = threadIdx.x & 31;
  const uint32_t lower_lanes = (1u << lane) - 1u;
  const int64_t nblk = uq_nblk(n);
  const int64_t tasks = nblk * k;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const bool vec = (((uintptr_t)models | (uintptr_t)theta | (uintptr_t)residual) & 15) == 0 && (model_stride & 3) == 0 &&
                   (residual_stride & 3) == 0 && (n & 3) == 0;
  for (int64_t t = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < tasks; t += warps) {
    const int c = (int)(t / nblk);
    const int64_t blk = t - (int64_t)c * nblk;
    const int64_t e0 = blk * kUqBlock + lane * 8;
    float* res = residual + c * residual_stride;
    float m[8], th[8], v[8];
    lane_load8<kLdStream>(models + c * model_stride, e0, n, vec, m);
    lane_load8<kLdReadOnly>(theta, e0, n, vec, th);
    lane_load8<kLdPlain>(res, e0, n, vec, v);
    TopkKeys8 keys;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      v[i] = (m[i] - th[i]) + v[i];
      keys.key[i] = (e0 + i < n) ? ut_key(v[i]) : 0u;
    }
    const TopkSel8 sel = warp_topk_select(keys, ut_block_k(n, blk, topk), lower_lanes);
    topk_emit(indices, values, c * entries + blk * topk, lane, sel, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = sel.keep[i] ? 0.f : v[i];
    lane_store8(res, e0, n, vec, v);
  }
}

// Sparse decode + FedAvg reduce + apply, the top-k twin of fedavg_q_kernel: one warp per 256-element block with a 256-float
// shared accumulator per warp.  Per slot in slot order, lanes < k_b scatter-fmaf their entry into it (a slot's offsets are
// distinct, and a __syncwarp separates slots: deterministic); the entries of 8 slots are loaded ahead of their scatters.  Then
// lane l reads elements 8 l .. 8 l + 7 back, a = theta + acc, and theta += opt.lr (a - theta) (OPT false) or the server
// optimizer step (OPT true).  A uint8 offset cannot leave the accumulator; offsets past the end of a partial last block land
// in accumulator cells no lane applies.
template <bool OPT>
__global__ void __launch_bounds__(256)
fedavg_topk_kernel(float* __restrict__ theta, const uint8_t* __restrict__ indices, const float* __restrict__ values, int64_t entries,
                   const float* __restrict__ weights, int k, int topk, ServerOptArgs opt, int64_t n) {
  constexpr int kAhead = 8;
  __shared__ float sw[StagedWeights::kSw];
  __shared__ __align__(16) float sacc[kThreads / 32][kUqBlock];
  const StagedWeights staged(sw, weights, k);
  const int lane = threadIdx.x & 31;
  float* acc = sacc[threadIdx.x >> 5];
  const int64_t nblk = uq_nblk(n);
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const bool vec = (((uintptr_t)theta | (uintptr_t)opt.m | (uintptr_t)opt.v) & 15) == 0;
  for (int64_t blk = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); blk < nblk; blk += warps) {
    const int64_t e0 = blk * kUqBlock + lane * 8;
    const int kb = ut_block_k(n, blk, topk);
    const bool sends = lane < kb;
    const int64_t slot0 = blk * topk + lane;
    *reinterpret_cast<float4*>(acc + lane * 8) = make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<float4*>(acc + lane * 8 + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncwarp();
    for (int c0 = 0; c0 < k; c0 += kAhead) {
      uint32_t idx[kAhead];
      float val[kAhead];
#pragma unroll
      for (int u = 0; u < kAhead; ++u) {
        idx[u] = 0;
        val[u] = 0.f;
        if (sends && c0 + u < k) {
          idx[u] = __ldcs(indices + (c0 + u) * entries + slot0);
          val[u] = __ldcs(values + (c0 + u) * entries + slot0);
        }
      }
#pragma unroll
      for (int u = 0; u < kAhead; ++u) {
        if (c0 + u < k) {
          if (sends) acc[idx[u]] = fmaf(staged.wt(c0 + u), val[u], acc[idx[u]]);
          __syncwarp();
        }
      }
    }
    if (e0 >= n) continue;
    float a8[8];
    const float4 lo = *reinterpret_cast<const float4*>(acc + lane * 8), hi = *reinterpret_cast<const float4*>(acc + lane * 8 + 4);
    a8[0] = lo.x; a8[1] = lo.y; a8[2] = lo.z; a8[3] = lo.w; a8[4] = hi.x; a8[5] = hi.y; a8[6] = hi.z; a8[7] = hi.w;
    apply8<OPT>(theta, e0, n, vec, a8, opt);
  }
}

// ---- compressed downlink (downlink.cuh) ---------------------------------------------------------------------------------------
// Coordinator, int8 / int4: quantize_delta_kernel's steps on d = theta - replica for one row, and the replica advanced in the
// same pass.
template <int BITS>
__global__ void __launch_bounds__(256)
downlink_quant_kernel(const float* __restrict__ theta, float* __restrict__ replica, uint32_t key, uint8_t* __restrict__ payload,
                      float* __restrict__ scales, int64_t n) {
  const int lane = threadIdx.x & 31;
  const int64_t nblk = uq_nblk(n);
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const bool vec = (((uintptr_t)theta | (uintptr_t)replica) & 15) == 0 && (n & 3) == 0;
  for (int64_t blk = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); blk < nblk; blk += warps) {
    const int64_t e0 = blk * kUqBlock + lane * 8;
    float t[8], r[8], d[8];
    lane_load8<kLdReadOnly>(theta, e0, n, vec, t);
    lane_load8<kLdPlain>(replica, e0, n, vec, r);
#pragma unroll
    for (int i = 0; i < 8; ++i) d[i] = t[i] - r[i];
    float step, inv;
    warp_block_scale<BITS>(d, step, inv);
    if (e0 < n) {
      int q[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        q[i] = uq_encode(d[i], inv, key, (uint32_t)(e0 + i), UqCodec<BITS>::kLevels);
        r[i] = dl_quant_advance(r[i], q[i], step);
      }
      store_codes8<BITS>(payload, e0, q);
      lane_store8(replica, e0, n, vec, r);
    }
    if (lane == 0) scales[blk] = step;
  }
}

// Coordinator, topk: the selection of topk_delta_kernel (warp_topk_select) on v = theta - replica with no residual; the kept
// entries go to the wire and are added into the replica (scalar stores of the kept elements only).
__global__ void __launch_bounds__(256)
downlink_topk_kernel(const float* __restrict__ theta, float* __restrict__ replica, int topk, uint8_t* __restrict__ indices,
                     float* __restrict__ values, int64_t n) {
  const int lane = threadIdx.x & 31;
  const uint32_t lower_lanes = (1u << lane) - 1u;
  const int64_t nblk = uq_nblk(n);
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const bool vec = (((uintptr_t)theta | (uintptr_t)replica) & 15) == 0 && (n & 3) == 0;
  for (int64_t blk = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); blk < nblk; blk += warps) {
    const int64_t e0 = blk * kUqBlock + lane * 8;
    float t[8], r[8], v[8];
    lane_load8<kLdReadOnly>(theta, e0, n, vec, t);
    lane_load8<kLdPlain>(replica, e0, n, vec, r);
    TopkKeys8 keys;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      v[i] = t[i] - r[i];
      keys.key[i] = (e0 + i < n) ? ut_key(v[i]) : 0u;
    }
    const TopkSel8 sel = warp_topk_select(keys, ut_block_k(n, blk, topk), lower_lanes);
    topk_emit(indices, values, blk * topk, lane, sel, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (sel.keep[i]) replica[e0 + i] = dl_add_rn(r[i], v[i]);
    }
  }
}

// Device, int8 / int4: replica += decode(wire), one warp per block.
template <int BITS>
__global__ void __launch_bounds__(256)
replica_apply_q_kernel(float* __restrict__ replica, const uint8_t* __restrict__ payload, const float* __restrict__ scales, int64_t n) {
  const int lane = threadIdx.x & 31;
  const int64_t nblk = uq_nblk(n);
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const bool vec = ((uintptr_t)replica & 15) == 0;
  for (int64_t blk = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); blk < nblk; blk += warps) {
    const int64_t e0 = blk * kUqBlock + lane * 8;
    if (e0 >= n) continue;
    const float step = __ldg(scales + blk);
    int q[8];
    load_codes8<BITS, kLdReadOnly>(payload, e0, q);
    // not lane_load8: this vec allows any n, so the groups of 4 inside n load 16 bytes and a last partial group scalars
    float r[8];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t e = e0 + 4 * h;
      if (vec && e + 4 <= n) {
        const float4 rp = *reinterpret_cast<const float4*>(replica + e);
        r[4 * h + 0] = rp.x; r[4 * h + 1] = rp.y; r[4 * h + 2] = rp.z; r[4 * h + 3] = rp.w;
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) r[4 * h + i] = e + i < n ? replica[e + i] : 0.f;
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) r[i] = dl_quant_advance(r[i], q[i], step);
    lane_store8(replica, e0, n, vec, r);
  }
}

// Device, topk: replica[j] += value for every entry, one warp per 256-element block, lane c < k_b taking entry c of the block
// (a block's offsets are distinct: no two lanes touch one element).  Offsets past n are skipped.
__global__ void __launch_bounds__(256)
replica_apply_topk_kernel(float* __restrict__ replica, const uint8_t* __restrict__ indices, const float* __restrict__ values, int topk,
                          int64_t n) {
  const int lane = threadIdx.x & 31;
  const int64_t nblk = uq_nblk(n);
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t blk = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); blk < nblk; blk += warps) {
    if (lane >= ut_block_k(n, blk, topk)) continue;
    const int64_t slot = blk * topk + lane;
    const int64_t j = blk * kUqBlock + __ldg(indices + slot);
    if (j < n) replica[j] = dl_add_rn(replica[j], __ldg(values + slot));
  }
}

// ---- secure aggregation (secagg.cuh) ------------------------------------------------------------------------------------------
// One thread per ChaCha20 column: column c is elements 16 c .. 16 c + 15, block c of every stream.  The 16 uint32 accumulators
// and one block of state stay in registers; a stream's key is the same for every thread of a launch at a given step (uniform
// 16-byte loads through the read-only cache: S can run into the thousands, the keys stay in global memory).

// the 16 words of column e0 of a uint32 row (0 past n): four 16-byte loads when `full`, scalar loads otherwise
template <LdHint HINT>
__device__ __forceinline__ void sa_load16(const uint32_t* __restrict__ p, int64_t e0, int64_t n, bool full, uint32_t (&x)[kSaWords]) {
  if (full) {
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const uint4 v = ld_hint<HINT>(reinterpret_cast<const uint4*>(p + e0) + h);
      x[4 * h + 0] = v.x; x[4 * h + 1] = v.y; x[4 * h + 2] = v.z; x[4 * h + 3] = v.w;
    }
  } else {
#pragma unroll
    for (int i = 0; i < kSaWords; ++i) x[i] = e0 + i < n ? p[e0 + i] : 0u;
  }
}

// acc += sum over the streams s0 <= s < s1 of signs[s] PRG(keys[s]), block `col`
__device__ __forceinline__ void sa_add_streams(uint32_t (&acc)[kSaWords], const uint32_t* __restrict__ keys, const int* __restrict__ signs,
                                               int s0, int s1, uint32_t col) {
#pragma unroll 1
  for (int s = s0; s < s1; ++s) {
    const uint4 lo = __ldg(reinterpret_cast<const uint4*>(keys + 8 * (int64_t)s));
    const uint4 hi = __ldg(reinterpret_cast<const uint4*>(keys + 8 * (int64_t)s) + 1);
    const uint32_t k[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    sa_add_block(acc, k, __ldg(signs + s), col);
  }
}

// Device: y = enc(model - theta) + sum_s signs[s] PRG(keys[s]) (mod 2^32), and the counts of clipped / non-finite deltas
// (counts[0] / counts[1], added to: the launcher zeroes them).
__global__ void __launch_bounds__(256)
secagg_mask_kernel(const float* __restrict__ model, const float* __restrict__ theta, const uint32_t* __restrict__ keys,
                   const int* __restrict__ signs, int streams, float clip, float scale, uint32_t* __restrict__ out, int* __restrict__ counts,
                   int64_t n) {
  const int64_t cols = (n + kSaWords - 1) / kSaWords;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const bool vec = (((uintptr_t)model | (uintptr_t)theta | (uintptr_t)out) & 15) == 0;
  int clipped = 0, nonfinite = 0;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < cols; c += stride) {
    const int64_t e0 = c * kSaWords;
    const bool full = vec && e0 + kSaWords <= n;
    uint32_t acc[kSaWords];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float m[8], t[8];
      lane_load8<kLdStream>(model, e0 + 8 * h, n, full, m);
      lane_load8<kLdReadOnly>(theta, e0 + 8 * h, n, full, t);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[8 * h + i] = sa_encode(m[i] - t[i], clip, scale, clipped, nonfinite);
    }
    sa_add_streams(acc, keys, signs, 0, streams, (uint32_t)c);
    if (full) {
#pragma unroll
      for (int h = 0; h < 4; ++h)
        reinterpret_cast<uint4*>(out + e0)[h] = make_uint4(acc[4 * h], acc[4 * h + 1], acc[4 * h + 2], acc[4 * h + 3]);
    } else {
#pragma unroll
      for (int i = 0; i < kSaWords; ++i) {
        if (e0 + i < n) out[e0 + i] = acc[i];
      }
    }
  }
  clipped = __reduce_add_sync(0xffffffffu, clipped);
  nonfinite = __reduce_add_sync(0xffffffffu, nonfinite);
  if ((threadIdx.x & 31) == 0) {
    if (clipped) atomicAdd(counts, clipped);
    if (nonfinite) atomicAdd(counts + 1, nonfinite);
  }
}

// Coordinator, split path (sa_streams_per_task > 0): task t = (chunk, column), per streams of the chunk expanded and added
// into partial[] (zeroed by the launcher) with atomicAdd.  Consecutive threads take consecutive columns of one chunk: the
// key loads stay uniform.
__global__ void __launch_bounds__(256)
secagg_streams_kernel(const uint32_t* __restrict__ keys, const int* __restrict__ signs, int streams, int per, uint32_t* __restrict__ partial,
                      int64_t n) {
  const int64_t cols = (n + kSaWords - 1) / kSaWords;
  const int64_t tasks = cols * ((streams + per - 1) / per);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < tasks; t += stride) {
    const int chunk = (int)(t / cols);
    const int64_t c = t - (int64_t)chunk * cols, e0 = c * kSaWords;
    const int s0 = chunk * per, s1 = s0 + per < streams ? s0 + per : streams;
    uint32_t acc[kSaWords];
#pragma unroll
    for (int i = 0; i < kSaWords; ++i) acc[i] = 0u;
    sa_add_streams(acc, keys, signs, s0, s1, (uint32_t)c);
#pragma unroll
    for (int i = 0; i < kSaWords; ++i) {
      if (e0 + i < n) atomicAdd(partial + e0 + i, acc[i]);
    }
  }
}

// Coordinator: z = sum of the k masked rows + the streams (all of them here when partial is null, else their sum from
// secagg_streams_kernel), mean = sa_decode(z), a = theta + mean, then theta += opt.lr (a - theta) (OPT false) or the server
// optimizer step (OPT true) through apply8.
template <bool OPT>
__global__ void __launch_bounds__(256)
fedavg_secagg_kernel(float* __restrict__ theta, const uint32_t* __restrict__ masked, int64_t row_stride, int k, const uint32_t* __restrict__ keys,
                     const int* __restrict__ signs, int streams, const uint32_t* __restrict__ partial, float inv_scale, float n_mean,
                     ServerOptArgs opt, int64_t n) {
  const int64_t cols = (n + kSaWords - 1) / kSaWords;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const bool vec_rows = (((uintptr_t)masked | (uintptr_t)partial) & 15) == 0 && (row_stride & 3) == 0;
  const bool vec = (((uintptr_t)theta | (uintptr_t)opt.m | (uintptr_t)opt.v) & 15) == 0;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < cols; c += stride) {
    const int64_t e0 = c * kSaWords;
    const bool full = vec_rows && e0 + kSaWords <= n;
    uint32_t acc[kSaWords];
    if (partial != nullptr) {
      sa_load16<kLdStream>(partial, e0, n, full, acc);
    } else {
#pragma unroll
      for (int i = 0; i < kSaWords; ++i) acc[i] = 0u;
      sa_add_streams(acc, keys, signs, 0, streams, (uint32_t)c);
    }
#pragma unroll 1
    for (int r = 0; r < k; ++r) {
      uint32_t y[kSaWords];
      sa_load16<kLdStream>(masked + r * row_stride, e0, n, full, y);
#pragma unroll
      for (int i = 0; i < kSaWords; ++i) acc[i] += y[i];
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mean[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) mean[i] = sa_decode(acc[8 * h + i], inv_scale, n_mean);
      apply8<OPT>(theta, e0 + 8 * h, n, vec, mean, opt);
    }
  }
}

// ---- losses ---------------------------------------------------------------------------------------
// the -100 floor of a BCE log term, as torch.clamp(min=-100) (and F.binary_cross_entropy) apply it: -inf becomes -100 and
// NaN stays NaN, so a diverged model reports a NaN loss (fmaxf(NaN, -100) would return -100)
__device__ __forceinline__ float bce_log_floor(float x) { return x < -100.f ? -100.f : x; }

__global__ void sigmoid_bce_kernel(const float* __restrict__ z, const float* __restrict__ y,
                                   float* __restrict__ dz, float* __restrict__ loss_out, int64_t n) {
  __shared__ float scratch[32];
  const float inv_n = 1.f / (float)n;
  float acc = 0.f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float p = 1.f / (1.f + __expf(-z[i]));
    const float t = y[i];
    const float lp = bce_log_floor(__logf(p)), l1p = bce_log_floor(log1pf(-p));
    acc -= t * lp + (1.f - t) * l1p;
    if (dz) dz[i] = (p - t) * inv_n;
  }
  acc = block_sum(acc, scratch);
  if (threadIdx.x == 0) atomicAdd(loss_out, acc * inv_n);
}

__global__ void sse_kernel(const float* __restrict__ out, const float* __restrict__ y,
                           float* __restrict__ dz, float* __restrict__ loss_out, int64_t n, float scale) {
  __shared__ float scratch[32];
  float acc = 0.f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float d = out[i] - y[i];
    acc = fmaf(d, d, acc);
    if (dz) dz[i] = 2.f * d * scale;
  }
  acc = block_sum(acc, scratch);
  if (threadIdx.x == 0) atomicAdd(loss_out, acc * scale);
}

// One warp per row; cols <= 1024.  Reads logits once, writes dlogits (fp32 and/or bf16).
template <bool BF16_IN>
__global__ void softmax_xent_kernel(const void* __restrict__ logits_, const int64_t* __restrict__ labels,
                                    float* __restrict__ dl, __nv_bfloat16* __restrict__ dl_bf16,
                                    float* __restrict__ loss_out, int rows, int cols) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const float inv_rows = 1.f / (float)rows;
  float loss_acc = 0.f;
  for (int r = blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < rows; r += gridDim.x * warps_per_block) {
    auto load = [&](int c) -> float {
      if (BF16_IN) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(logits_)[(size_t)r * cols + c]);
      return reinterpret_cast<const float*>(logits_)[(size_t)r * cols + c];
    };
    float m = -INFINITY;
    for (int c = lane; c < cols; c += 32) m = fmaxf(m, load(c));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int c = lane; c < cols; c += 32) s += __expf(load(c) - m);
    s = warp_sum(s);
    const int label = (int)labels[r];
    const float inv_s = 1.f / s;
    for (int c = lane; c < cols; c += 32) {
      const float z = load(c);
      const float g = (__expf(z - m) * inv_s - (c == label ? 1.f : 0.f)) * inv_rows;
      if (dl) dl[(size_t)r * cols + c] = g;
      if (dl_bf16) dl_bf16[(size_t)r * cols + c] = __float2bfloat16(g);
      if (c == label) loss_acc += (__logf(s) + m) - z;
    }
  }
  loss_acc = warp_sum(loss_acc);
  if (lane == 0 && loss_acc != 0.f) atomicAdd(loss_out, loss_acc * inv_rows);
}

// Loss head of the GEMM-shaped trainers in ONE launch and ONE block: softmax cross-entropy of the valid rows / columns of a PADDED
// fp32 (or bf16) logits matrix, dL/dlogits written straight into the padded bf16 operand of the backward GEMMs (and / or an fp32
// matrix), the head's bias gradient (column sums of dL/dlogits) and the mean loss.  Replaces slice-copy + loss + cast-copy +
// at::sum + copy (three ATen launches, one of them a single-block reduction) around the old kernel.  One block, fixed
// summation order: bit-reproducible, no memset, no atomics.  cols <= kHeadMaxCols.
constexpr int kHeadMaxCols = 128;
template <bool BF16_IN>
__global__ void __launch_bounds__(1024)
softmax_xent_head_kernel(const void* __restrict__ logits_, int ld_in, const int64_t* __restrict__ labels, float* __restrict__ dl, int ld_dl,
                         __nv_bfloat16* __restrict__ dl_bf16, int ld_bf16, float* __restrict__ db, float* __restrict__ loss_out, int rows,
                         int cols) {
  __shared__ float s_col[32][kHeadMaxCols + 1];
  __shared__ float s_loss[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const float inv_rows = 1.f / (float)rows;
  float colacc[kHeadMaxCols / 32];
#pragma unroll
  for (int j = 0; j < kHeadMaxCols / 32; ++j) colacc[j] = 0.f;
  float loss_acc = 0.f;
  for (int r = warp; r < rows; r += nwarps) {
    auto load = [&](int c) -> float {
      if (BF16_IN) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(logits_)[(size_t)r * ld_in + c]);
      return reinterpret_cast<const float*>(logits_)[(size_t)r * ld_in + c];
    };
    float z[kHeadMaxCols / 32];
    float m = -INFINITY;
#pragma unroll
    for (int j = 0; j < kHeadMaxCols / 32; ++j) {
      const int c = lane + 32 * j;
      z[j] = c < cols ? load(c) : -INFINITY;
      m = fmaxf(m, z[j]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < kHeadMaxCols / 32; ++j)
      if (lane + 32 * j < cols) s += __expf(z[j] - m);
    s = warp_sum(s);
    const int label = (int)labels[r];
    const float inv_s = 1.f / s;
#pragma unroll
    for (int j = 0; j < kHeadMaxCols / 32; ++j) {
      const int c = lane + 32 * j;
      if (c < cols) {
        const float g = (__expf(z[j] - m) * inv_s - (c == label ? 1.f : 0.f)) * inv_rows;
        if (dl) dl[(size_t)r * ld_dl + c] = g;
        if (dl_bf16) dl_bf16[(size_t)r * ld_bf16 + c] = __float2bfloat16(g);
        colacc[j] += g;
        if (c == label) loss_acc += (__logf(s) + m) - z[j];
      }
    }
  }
#pragma unroll
  for (int j = 0; j < kHeadMaxCols / 32; ++j) s_col[warp][lane + 32 * j] = colacc[j];
  loss_acc = warp_sum(loss_acc);
  if (lane == 0) s_loss[warp] = loss_acc;
  __syncthreads();
  if (db) {
    for (int c = threadIdx.x; c < cols; c += blockDim.x) {
      float t = 0.f;
      for (int w = 0; w < nwarps; ++w) t += s_col[w][c];
      db[c] = t;
    }
  }
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < nwarps; ++w) t += s_loss[w];
    *loss_out = t * inv_rows;
  }
}

__global__ void eval_binary_kernel(const float* __restrict__ p, const float* __restrict__ y,
                                   float* __restrict__ loss_sum, int* __restrict__ correct, int64_t n) {
  __shared__ float scratch[32];
  float acc = 0.f;
  int ok = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float q = p[i], t = y[i];
    const float lp = bce_log_floor(__logf(q)), l1p = bce_log_floor(log1pf(-q));
    acc -= t * lp + (1.f - t) * l1p;
    ok += (rintf(q) == t) ? 1 : 0;
  }
  acc = block_sum(acc, scratch);
  if (threadIdx.x == 0) atomicAdd(loss_sum, acc);
  ok = __reduce_add_sync(0xffffffffu, ok);
  if ((threadIdx.x & 31) == 0 && ok) atomicAdd(correct, ok);
}

// torch.argmax order: NaN above every number, the lowest index among equals (among NaNs too, which is what keeps the rule
// across the lanes of the shuffle merge)
__device__ __forceinline__ bool argmax_takes(float v, int c, float best, int bi) {
  return isnan(v) ? (!isnan(best) || c < bi) : (v > best || (v == best && c < bi));
}

__global__ void argmax_rows_kernel(const float* __restrict__ x, int64_t* __restrict__ out, int rows, int cols) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < rows; r += gridDim.x * wpb) {
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = lane; c < cols; c += 32) {
      const float v = x[(size_t)r * cols + c];
      if (argmax_takes(v, c, best, bi)) { best = v; bi = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (argmax_takes(ov, oi, best, bi)) { best = ov; bi = oi; }
    }
    if (lane == 0) out[r] = bi;
  }
}

// MinMax: one block per column pass 1 (min/max), pass 2 scale.  cols is tiny (10).
__global__ void minmax_scale_kernel(const float* __restrict__ x, float* __restrict__ out, int rows, int cols) {
  __shared__ float smin[32], smax[32];
  const int c = blockIdx.x;
  float lo = INFINITY, hi = -INFINITY;
  for (int r = threadIdx.x; r < rows; r += blockDim.x) {
    const float v = x[(size_t)r * cols + c];
    lo = fminf(lo, v); hi = fmaxf(hi, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { smin[w] = lo; smax[w] = hi; }
  __syncthreads();
  lo = smin[0]; hi = smax[0];
  for (int i = 1; i < (blockDim.x >> 5); ++i) { lo = fminf(lo, smin[i]); hi = fmaxf(hi, smax[i]); }
  float rng = hi - lo;
  if (rng == 0.f) rng = 1.f;
  const float inv = 1.f / rng;
  for (int r = threadIdx.x; r < rows; r += blockDim.x)
    out[(size_t)r * cols + c] = (x[(size_t)r * cols + c] - lo) * inv;
}

// Keyed random permutations, one row per epoch (the bijection itself: feistel_index in colearn_kernels.h)
__global__ void feistel_perm_kernel(int* __restrict__ out, int n, int rows, uint64_t seed) {
  const FeistelDomain dom = feistel_domain((uint32_t)n);
  const int64_t total = (int64_t)n * rows;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
    const int row = (int)(e / n);
    out[e] = (int)feistel_index((uint32_t)(e - (int64_t)row * n), (uint32_t)n, dom, seed, row);
  }
}

__global__ void fp32_to_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (((((uintptr_t)in) & 15) == 0) && ((((uintptr_t)out) & 7) == 0)) {
    const int64_t n4 = n >> 2;
    for (int64_t j = i0; j < n4; j += stride) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(in) + j);
      __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
      uint2 pk;
      pk.x = *reinterpret_cast<uint32_t*>(&a);
      pk.y = *reinterpret_cast<uint32_t*>(&b);
      reinterpret_cast<uint2*>(out)[j] = pk;
    }
    for (int64_t j = (n4 << 2) + i0; j < n; j += stride) out[j] = __float2bfloat16(in[j]);
  } else {
    for (int64_t j = i0; j < n; j += stride) out[j] = __float2bfloat16(in[j]);
  }
}

__global__ void transpose_bf16_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int rows, int cols) {
  __shared__ __nv_bfloat16 tile[32][34];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int r = r0 + j, c = c0 + threadIdx.x;
    if (r < rows && c < cols) tile[j][threadIdx.x] = in[(size_t)r * cols + c];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (r < rows && c < cols) out[(size_t)c * rows + r] = tile[threadIdx.x][j];
  }
}

// ---- int64 ring ops for the SMPC path (SURVEY K18): Z_{2^64} arithmetic on CUDA cores ---------------------
__global__ void fix_precision_kernel(const float* __restrict__ x, long long* __restrict__ out, int64_t n, double base) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    out[i] = (long long)rint((double)x[i] * base);   // round-half-even, same as torch.round
}
__global__ void float_precision_kernel(const long long* __restrict__ x, float* __restrict__ out, int64_t n, double inv_base) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    out[i] = (float)((double)x[i] * inv_base);
}
// C[m,n] = sum_k A[m,k] * B[k,n]  (mod 2^64; unsigned wrap-around == two's complement ring arithmetic)
__global__ void ring_matmul_kernel(const unsigned long long* __restrict__ A, const unsigned long long* __restrict__ B,
                                   unsigned long long* __restrict__ C, int M, int K, int N) {
  __shared__ unsigned long long sa[16][17], sb[16][17];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int row = blockIdx.y * 16 + ty, col = blockIdx.x * 16 + tx;
  unsigned long long acc = 0ull;
  for (int k0 = 0; k0 < K; k0 += 16) {
    sa[ty][tx] = (row < M && k0 + tx < K) ? A[(size_t)row * K + k0 + tx] : 0ull;
    sb[ty][tx] = (k0 + ty < K && col < N) ? B[(size_t)(k0 + ty) * N + col] : 0ull;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) acc += sa[ty][k] * sb[k][tx];
    __syncthreads();
  }
  if (row < M && col < N) C[(size_t)row * N + col] = acc;
}

__global__ void bias_sgd_from_partials_kernel(float* __restrict__ bias, const float* __restrict__ partials, int rows, int n,
                                              int64_t row_stride, float lr, float* __restrict__ grad_out, int n_bias) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n) return;
  float g = 0.f;
  for (int r = 0; r < rows; ++r) g += partials[(size_t)r * row_stride + c];
  if (grad_out) grad_out[c] = g;
  if (bias && c < n_bias) bias[c] = fmaf(-lr, g, bias[c]);
}

__global__ void l2_flush_kernel(float* __restrict__ buf, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) buf[i] = (float)i;
}

}  // namespace

cudaError_t launch_sgd_step(float* p, const float* g, float lr, int64_t n, cudaStream_t s) {
  COLEARN_LAUNCH(sgd_step_kernel, grid_for(n), kThreads, 0, s, p, g, lr, n);
  return cudaGetLastError();
}
cudaError_t launch_scale_inplace(float* p, float scale, int64_t n, cudaStream_t s) {
  COLEARN_LAUNCH(scale_inplace_kernel, grid_for(n), kThreads, 0, s, p, scale, n);
  return cudaGetLastError();
}
cudaError_t launch_sgd_step_bf16grad(float* p, const void* g, float lr, int64_t n, cudaStream_t s) {
  COLEARN_LAUNCH(sgd_step_bf16grad_kernel, grid_for(n), kThreads, 0, s, p, reinterpret_cast<const __nv_bfloat16*>(g), lr, n);
  return cudaGetLastError();
}
cudaError_t launch_fedavg_apply(float* theta, const float* slots, int64_t slot_stride, const float* weights,
                                int k, float server_lr, int64_t n, cudaStream_t s) {
  if (k < 1) return cudaErrorInvalidValue;
  COLEARN_LAUNCH(fedavg_kernel<true>, grid_for(n), kThreads, 0, s, theta, slots, slot_stride, weights, k, server_lr, n);
  return cudaGetLastError();
}
cudaError_t launch_fedavg_apply_opt(float* theta, const float* slots, int64_t slot_stride, const float* weights, int k,
                                    const ServerOptArgs& opt, int64_t n, cudaStream_t s) {
  if (k < 1 || !server_opt_args_ok(opt)) return cudaErrorInvalidValue;
  if (opt.kind == SOPT_SGD) return launch_fedavg_apply(theta, slots, slot_stride, weights, k, opt.lr, n, s);
  COLEARN_LAUNCH(fedavg_opt_kernel, grid_for(n), kThreads, 0, s, theta, slots, slot_stride, weights, k, opt, n);
  return cudaGetLastError();
}
cudaError_t launch_fedavg_apply_robust(float* theta, const float* slots, int64_t slot_stride, int k, const AggArgs& agg,
                                       const ServerOptArgs& opt, int64_t n, cudaStream_t s) {
  if (k < 1 || agg.kind == AGG_MEAN || !agg_args_ok(agg) || !server_opt_args_ok(opt)) return cudaErrorInvalidValue;
  const int grid = grid_for(n, 1);
  // the register path costs KMAX^2 compares per element whatever k is: take the smallest that holds k
  if (k <= 4) {
    COLEARN_LAUNCH(fedavg_robust_kernel<4>, grid, kThreads, 0, s, theta, slots, slot_stride, k, agg, opt, n);
  } else if (k <= 8) {
    COLEARN_LAUNCH(fedavg_robust_kernel<8>, grid, kThreads, 0, s, theta, slots, slot_stride, k, agg, opt, n);
  } else if (k <= 16) {
    COLEARN_LAUNCH(fedavg_robust_kernel<16>, grid, kThreads, 0, s, theta, slots, slot_stride, k, agg, opt, n);
  } else if (k <= 32) {
    COLEARN_LAUNCH(fedavg_robust_kernel<32>, grid, kThreads, 0, s, theta, slots, slot_stride, k, agg, opt, n);
  } else {
    COLEARN_LAUNCH(fedavg_robust_kernel<0>, grid, kThreads, 0, s, theta, slots, slot_stride, k, agg, opt, n);
  }
  return cudaGetLastError();
}
namespace {
// one warp per 256-element block (of one row): 8 warps per CTA, at most the persistent grid
inline int grid_for_warps(int64_t warp_tasks) {
  int64_t b = (warp_tasks + kThreads / 32 - 1) / (kThreads / 32);
  if (b > 132 * 8) b = 132 * 8;
  return (int)(b < 1 ? 1 : b);
}
// kernel pointers: launched through COLEARN_LAUNCH like a kernel name (template argument lists would split the macro's arguments)
template <int BITS>
inline cudaError_t launch_quantize_delta_t(const float* models, int64_t model_stride, const float* theta, const uint32_t* keys, int k,
                                           uint8_t* payload, int64_t row_bytes, float* scales, int64_t n, cudaStream_t s) {
  auto kernel = quantize_delta_kernel<BITS>;
  COLEARN_LAUNCH(kernel, grid_for_warps(k * uq_nblk(n)), kThreads, 0, s, models, model_stride, theta, keys, k, payload,
                 row_bytes, scales, n);
  return cudaGetLastError();
}
template <int BITS>
inline cudaError_t launch_fedavg_q_t(float* theta, const uint8_t* payload, int64_t row_bytes, const float* scales, const float* weights,
                                     int k, const ServerOptArgs& opt, int64_t n, cudaStream_t s) {
  const int grid = grid_for_warps(uq_nblk(n));
  if (opt.kind == SOPT_SGD) {
    auto kernel = fedavg_q_kernel<BITS, false>;
    COLEARN_LAUNCH(kernel, grid, kThreads, 0, s, theta, payload, row_bytes, scales, weights, k, opt, n);
  } else {
    auto kernel = fedavg_q_kernel<BITS, true>;
    COLEARN_LAUNCH(kernel, grid, kThreads, 0, s, theta, payload, row_bytes, scales, weights, k, opt, n);
  }
  return cudaGetLastError();
}
template <int BITS>
inline cudaError_t launch_fedavg_q_robust_t(float* theta, const uint8_t* payload, int64_t row_bytes, const float* scales, int k,
                                            const AggArgs& agg, const ServerOptArgs& opt, int64_t n, cudaStream_t s) {
  const int grid = grid_for(n, 1);
  void (*kernel)(float*, const uint8_t*, int64_t, const float*, int, AggArgs, ServerOptArgs, int64_t);
  // as launch_fedavg_apply_robust: the smallest register path that holds k, the general path above 32
  if (k <= 4) kernel = fedavg_q_robust_kernel<4, BITS>;
  else if (k <= 8) kernel = fedavg_q_robust_kernel<8, BITS>;
  else if (k <= 16) kernel = fedavg_q_robust_kernel<16, BITS>;
  else if (k <= 32) kernel = fedavg_q_robust_kernel<32, BITS>;
  else kernel = fedavg_q_robust_kernel<0, BITS>;
  COLEARN_LAUNCH(kernel, grid, kThreads, 0, s, theta, payload, row_bytes, scales, k, agg, opt, n);
  return cudaGetLastError();
}
inline bool uq_layout_ok(int bits, const uint8_t* payload, int64_t row_bytes, int64_t n) {
  if (bits != 8 && bits != 4) return false;
  if (n < 1 || n >= ((int64_t)1 << 31)) return false;            // element indices are hashed as uint32
  const int64_t need = bits == 8 ? n : (n + 1) / 2;
  return (row_bytes & 15) == 0 && row_bytes >= need && (reinterpret_cast<uintptr_t>(payload) & 15) == 0;
}
}  // namespace

cudaError_t launch_quantize_delta(const float* models, int64_t model_stride, const float* theta, const uint32_t* keys, int k, int bits,
                                  uint8_t* payload, int64_t row_bytes, float* scales, int64_t n, cudaStream_t s) {
  if (k < 1 || model_stride < n || !uq_layout_ok(bits, payload, row_bytes, n)) return cudaErrorInvalidValue;
  return bits == 8 ? launch_quantize_delta_t<8>(models, model_stride, theta, keys, k, payload, row_bytes, scales, n, s)
                   : launch_quantize_delta_t<4>(models, model_stride, theta, keys, k, payload, row_bytes, scales, n, s);
}
cudaError_t launch_fedavg_apply_quantized(float* theta, const uint8_t* payload, int64_t row_bytes, const float* scales,
                                          const float* weights, int k, int bits, const ServerOptArgs& opt, int64_t n, cudaStream_t s) {
  if (k < 1 || !uq_layout_ok(bits, payload, row_bytes, n) || !server_opt_args_ok(opt)) return cudaErrorInvalidValue;
  return bits == 8 ? launch_fedavg_q_t<8>(theta, payload, row_bytes, scales, weights, k, opt, n, s)
                   : launch_fedavg_q_t<4>(theta, payload, row_bytes, scales, weights, k, opt, n, s);
}
cudaError_t launch_fedavg_apply_quantized_robust(float* theta, const uint8_t* payload, int64_t row_bytes, const float* scales, int k,
                                                 int bits, const AggArgs& agg, const ServerOptArgs& opt, int64_t n, cudaStream_t s) {
  if (k < 1 || agg.kind == AGG_MEAN || !agg_args_ok(agg) || !server_opt_args_ok(opt) || !uq_layout_ok(bits, payload, row_bytes, n))
    return cudaErrorInvalidValue;
  return bits == 8 ? launch_fedavg_q_robust_t<8>(theta, payload, row_bytes, scales, k, agg, opt, n, s)
                   : launch_fedavg_q_robust_t<4>(theta, payload, row_bytes, scales, k, agg, opt, n, s);
}
namespace {
// The passes of one distance-based aggregation: the distance pass, its finalisation, then per geomed step l < L the fused centre
// + distance pass and its finalisation, and the apply pass: 2 L + 1 launches (norm_clip: 3).  grid <= 0: one CTA per chunk up to
// the persistent grid.
template <class Rows, bool CLIP, bool OPT>
inline void launch_dagg_apply_t(Rows rows, float* theta, int k, const DistAggScratch& sc, const ServerOptArgs& opt, int64_t n, int grid,
                                cudaStream_t s) {
  auto kernel = dagg_apply_kernel<Rows, CLIP, OPT>;
  COLEARN_LAUNCH(kernel, grid, kDaThreads, 0, s, rows, theta, k, sc, opt, n);
}
template <class Rows>
inline cudaError_t launch_dagg_t(const Rows& rows, float* theta, const float* alpha, int k, const DistAggArgs& g, const ServerOptArgs& opt,
                                 int64_t n, void* scratch, float* w_out, int grid, cudaStream_t s) {
  const int64_t nchunks = da_chunks(n);
  if (grid <= 0) grid = (int)(nchunks < 132 * 8 ? nchunks : 132 * 8);
  const DistAggScratch sc = da_scratch_carve(scratch, k, n);
  cudaError_t e = cudaMemsetAsync(sc.ticket, 0, sizeof(unsigned), s);
  if (e != cudaSuccess) return e;
  {
    auto kernel = dagg_dist_kernel<Rows>;
    COLEARN_LAUNCH(kernel, grid, kDaThreads, 0, s, rows, theta, k, sc, n);
  }
  COLEARN_LAUNCH(dagg_finalize_kernel, k, kDaThreads, 0, s, sc, alpha, k, g, w_out, nchunks);
  const int steps = g.kind == DAGG_GEOMED ? g.iters - 1 : 0;
  for (int l = 0; l < steps; ++l) {
    void (*kernel)(Rows, const float*, int, DistAggScratch, int64_t);
    // the register path holds 8 KMAX floats of rows per lane: KMAX 16 is the largest that stays clear of spills
    if (k <= 4) kernel = dagg_center_kernel<4, Rows>;
    else if (k <= 8) kernel = dagg_center_kernel<8, Rows>;
    else if (k <= 16) kernel = dagg_center_kernel<16, Rows>;
    else kernel = dagg_center_kernel<0, Rows>;
    COLEARN_LAUNCH(kernel, grid, kDaThreads, 0, s, rows, theta, k, sc, n);
    COLEARN_LAUNCH(dagg_finalize_kernel, k, kDaThreads, 0, s, sc, alpha, k, g, w_out, nchunks);
  }
  const bool clip = g.kind == DAGG_NORM_CLIP, o = opt.kind != SOPT_SGD;
  if (clip && o) launch_dagg_apply_t<Rows, true, true>(rows, theta, k, sc, opt, n, grid, s);
  else if (clip) launch_dagg_apply_t<Rows, true, false>(rows, theta, k, sc, opt, n, grid, s);
  else if (o) launch_dagg_apply_t<Rows, false, true>(rows, theta, k, sc, opt, n, grid, s);
  else launch_dagg_apply_t<Rows, false, false>(rows, theta, k, sc, opt, n, grid, s);
  return cudaGetLastError();
}
inline bool dagg_ok(int k, const DistAggArgs& g, const ServerOptArgs& opt, int64_t n, const void* scratch) {
  return k >= 1 && n >= 1 && dist_agg_args_ok(g) && server_opt_args_ok(opt) && scratch != nullptr &&
         (reinterpret_cast<uintptr_t>(scratch) & 15) == 0;
}
}  // namespace

cudaError_t launch_fedavg_apply_distance(float* theta, const float* rows, int64_t row_stride, const float* weights, int k,
                                         const DistAggArgs& g, const ServerOptArgs& opt, int64_t n, void* scratch, float* weights_out,
                                         int grid, cudaStream_t s) {
  if (!dagg_ok(k, g, opt, n, scratch) || row_stride < n) return cudaErrorInvalidValue;
  const bool vec = ((uintptr_t)rows & 15) == 0 && (row_stride & 3) == 0 && (n & 3) == 0;
  return launch_dagg_t(F32Rows{rows, row_stride, n, vec}, theta, weights, k, g, opt, n, scratch, weights_out, grid, s);
}
cudaError_t launch_fedavg_apply_quantized_distance(float* theta, const uint8_t* payload, int64_t row_bytes, const float* scales,
                                                   const float* weights, int k, int bits, const DistAggArgs& g, const ServerOptArgs& opt,
                                                   int64_t n, void* scratch, float* weights_out, int grid, cudaStream_t s) {
  if (!dagg_ok(k, g, opt, n, scratch) || !uq_layout_ok(bits, payload, row_bytes, n)) return cudaErrorInvalidValue;
  if (bits == 8) return launch_dagg_t(QRows<8>{payload, row_bytes, scales, uq_nblk(n), n}, theta, weights, k, g, opt, n, scratch, weights_out, grid, s);
  return launch_dagg_t(QRows<4>{payload, row_bytes, scales, uq_nblk(n), n}, theta, weights, k, g, opt, n, scratch, weights_out, grid, s);
}
cudaError_t launch_topk_delta(const float* models, int64_t model_stride, const float* theta, float* residual, int64_t residual_stride,
                              int rows, int topk, uint8_t* indices, float* values, int64_t entries, int64_t n, cudaStream_t s) {
  if (rows < 1 || topk < 1 || topk > kUtMaxK || n < 1 || model_stride < n || residual_stride < n || entries < ut_entries(n, topk))
    return cudaErrorInvalidValue;
  COLEARN_LAUNCH(topk_delta_kernel, grid_for_warps(rows * uq_nblk(n)), kThreads, 0, s, models, model_stride, theta,
                 residual, residual_stride, rows, topk, indices, values, entries, n);
  return cudaGetLastError();
}
cudaError_t launch_fedavg_apply_topk(float* theta, const uint8_t* indices, const float* values, int64_t entries, const float* weights,
                                     int rows, int topk, const ServerOptArgs& opt, int64_t n, cudaStream_t s) {
  if (rows < 1 || topk < 1 || topk > kUtMaxK || n < 1 || entries < ut_entries(n, topk) || !server_opt_args_ok(opt))
    return cudaErrorInvalidValue;
  const int grid = grid_for_warps(uq_nblk(n));
  if (opt.kind == SOPT_SGD) {
    COLEARN_LAUNCH(fedavg_topk_kernel<false>, grid, kThreads, 0, s, theta, indices, values, entries, weights, rows, topk, opt, n);
  } else {
    COLEARN_LAUNCH(fedavg_topk_kernel<true>, grid, kThreads, 0, s, theta, indices, values, entries, weights, rows, topk, opt, n);
  }
  return cudaGetLastError();
}
cudaError_t launch_downlink_quant(const float* theta, float* replica, uint32_t key, int bits, uint8_t* payload, int64_t row_bytes,
                                  float* scales, int64_t n, cudaStream_t s) {
  if (!uq_layout_ok(bits, payload, row_bytes, n)) return cudaErrorInvalidValue;
  auto kernel = bits == 8 ? downlink_quant_kernel<8> : downlink_quant_kernel<4>;
  COLEARN_LAUNCH(kernel, grid_for_warps(uq_nblk(n)), kThreads, 0, s, theta, replica, key, payload, scales, n);
  return cudaGetLastError();
}
cudaError_t launch_downlink_topk(const float* theta, float* replica, int topk, uint8_t* indices, float* values, int64_t n, cudaStream_t s) {
  if (topk < 1 || topk > kUtMaxK || n < 1) return cudaErrorInvalidValue;
  COLEARN_LAUNCH(downlink_topk_kernel, grid_for_warps(uq_nblk(n)), kThreads, 0, s, theta, replica, topk, indices,
                 values, n);
  return cudaGetLastError();
}
cudaError_t launch_replica_apply_quant(float* replica, const uint8_t* payload, int64_t row_bytes, const float* scales, int bits,
                                       int64_t n, cudaStream_t s) {
  if (!uq_layout_ok(bits, payload, row_bytes, n)) return cudaErrorInvalidValue;
  auto kernel = bits == 8 ? replica_apply_q_kernel<8> : replica_apply_q_kernel<4>;
  COLEARN_LAUNCH(kernel, grid_for_warps(uq_nblk(n)), kThreads, 0, s, replica, payload, scales, n);
  return cudaGetLastError();
}
cudaError_t launch_replica_apply_topk(float* replica, const uint8_t* indices, const float* values, int topk, int64_t n, cudaStream_t s) {
  if (topk < 1 || topk > kUtMaxK || n < 1) return cudaErrorInvalidValue;
  COLEARN_LAUNCH(replica_apply_topk_kernel, grid_for_warps(uq_nblk(n)), kThreads, 0, s, replica, indices, values,
                 topk, n);
  return cudaGetLastError();
}
cudaError_t launch_secagg_mask(const float* model, const float* theta, const uint32_t* keys, const int* signs, int streams, float clip,
                               int frac_bits, uint32_t* out, int* counts, int64_t n, cudaStream_t s) {
  if (n < 1 || n >= kSaMaxElems || streams < 0 || !(clip > 0.f) || !(clip < INFINITY) || frac_bits < 0 || frac_bits > 64 ||
      (reinterpret_cast<uintptr_t>(keys) & 15) != 0)
    return cudaErrorInvalidValue;
  cudaError_t e = cudaMemsetAsync(counts, 0, 2 * sizeof(int), s);
  if (e != cudaSuccess) return e;
  COLEARN_LAUNCH(secagg_mask_kernel, grid_for((n + kSaWords - 1) / kSaWords, 1), kThreads, 0, s, model, theta, keys, signs, streams, clip,
                 ldexpf(1.f, frac_bits), out, counts, n);
  return cudaGetLastError();
}
cudaError_t launch_fedavg_apply_secagg(float* theta, const uint32_t* masked, int64_t row_stride, int k, const uint32_t* keys, const int* signs,
                                       int streams, uint32_t* workspace, int frac_bits, int n_mean, const ServerOptArgs& opt, int64_t n,
                                       cudaStream_t s) {
  if (k < 1 || n < 1 || n >= kSaMaxElems || row_stride < n || streams < 0 || n_mean < 1 || frac_bits < 0 || frac_bits > 64 ||
      (reinterpret_cast<uintptr_t>(keys) & 15) != 0 || !server_opt_args_ok(opt))
    return cudaErrorInvalidValue;
  const int64_t cols = (n + kSaWords - 1) / kSaWords;
  const int per = sa_streams_per_task(n, streams);
  const uint32_t* partial = nullptr;
  if (per > 0) {
    if (workspace == nullptr) return cudaErrorInvalidValue;
    cudaError_t e = cudaMemsetAsync(workspace, 0, (size_t)n * sizeof(uint32_t), s);
    if (e != cudaSuccess) return e;
    COLEARN_LAUNCH(secagg_streams_kernel, grid_for(cols * ((streams + per - 1) / per), 1), kThreads, 0, s, keys, signs, streams, per,
                   workspace, n);
    partial = workspace;
  }
  const float inv_scale = ldexpf(1.f, -frac_bits), nf = (float)n_mean;
  if (opt.kind == SOPT_SGD) {
    COLEARN_LAUNCH(fedavg_secagg_kernel<false>, grid_for(cols, 1), kThreads, 0, s, theta, masked, row_stride, k, keys, signs, streams,
                   partial, inv_scale, nf, opt, n);
  } else {
    COLEARN_LAUNCH(fedavg_secagg_kernel<true>, grid_for(cols, 1), kThreads, 0, s, theta, masked, row_stride, k, keys, signs, streams,
                   partial, inv_scale, nf, opt, n);
  }
  return cudaGetLastError();
}
cudaError_t launch_fedavg_flat(float* out, const float* slots, int64_t slot_stride, const float* weights,
                               int k, int64_t n, cudaStream_t s) {
  if (k < 1) return cudaErrorInvalidValue;
  COLEARN_LAUNCH(fedavg_kernel<false>, grid_for(n), kThreads, 0, s, out, slots, slot_stride, weights, k, 1.f, n);
  return cudaGetLastError();
}
cudaError_t launch_sigmoid_bce(const float* z, const float* y, float* dz, float* loss_out, int64_t n, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(loss_out, 0, sizeof(float), s);
  if (e != cudaSuccess) return e;
  COLEARN_LAUNCH(sigmoid_bce_kernel, grid_for(n, 1), kThreads, 0, s, z, y, dz, loss_out, n);
  return cudaGetLastError();
}
cudaError_t launch_sse(const float* out, const float* y, float* dz, float* loss_out, int64_t n, float scale, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(loss_out, 0, sizeof(float), s);
  if (e != cudaSuccess) return e;
  COLEARN_LAUNCH(sse_kernel, grid_for(n, 1), kThreads, 0, s, out, y, dz, loss_out, n, scale);
  return cudaGetLastError();
}
cudaError_t launch_softmax_xent(const void* logits, int is_bf16, const int64_t* labels, float* dl, void* dl_bf16,
                                float* loss_out, int rows, int cols, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(loss_out, 0, sizeof(float), s);
  if (e != cudaSuccess) return e;
  const int wpb = kThreads / 32;
  int blocks = (rows + wpb - 1) / wpb;
  if (blocks > 132 * 8) blocks = 132 * 8;
  if (blocks < 1) blocks = 1;
  if (is_bf16)
    COLEARN_LAUNCH(softmax_xent_kernel<true>, blocks, kThreads, 0, s, logits, labels, dl, reinterpret_cast<__nv_bfloat16*>(dl_bf16), loss_out, rows, cols);
  else
    COLEARN_LAUNCH(softmax_xent_kernel<false>, blocks, kThreads, 0, s, logits, labels, dl, reinterpret_cast<__nv_bfloat16*>(dl_bf16), loss_out, rows, cols);
  return cudaGetLastError();
}
cudaError_t launch_softmax_xent_head(const void* logits, int is_bf16, int ld_in, const int64_t* labels, float* dl, int ld_dl, void* dl_bf16,
                                     int ld_bf16, float* db, float* loss_out, int rows, int cols, cudaStream_t s) {
  if (cols < 1 || cols > kHeadMaxCols || rows < 1) return cudaErrorInvalidValue;
  int threads = 32 * (rows < 32 ? rows : 32);          // one warp per row in flight, at most 32 warps
  if (is_bf16)
    COLEARN_LAUNCH(softmax_xent_head_kernel<true>, 1, threads, 0, s, logits, ld_in, labels, dl, ld_dl, reinterpret_cast<__nv_bfloat16*>(dl_bf16),
                   ld_bf16, db, loss_out, rows, cols);
  else
    COLEARN_LAUNCH(softmax_xent_head_kernel<false>, 1, threads, 0, s, logits, ld_in, labels, dl, ld_dl, reinterpret_cast<__nv_bfloat16*>(dl_bf16),
                   ld_bf16, db, loss_out, rows, cols);
  return cudaGetLastError();
}
cudaError_t launch_eval_binary(const float* p, const float* y, float* loss_sum, int* correct, int64_t n, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(loss_sum, 0, sizeof(float), s);
  if (e != cudaSuccess) return e;
  e = cudaMemsetAsync(correct, 0, sizeof(int), s);
  if (e != cudaSuccess) return e;
  COLEARN_LAUNCH(eval_binary_kernel, grid_for(n, 1), kThreads, 0, s, p, y, loss_sum, correct, n);
  return cudaGetLastError();
}
cudaError_t launch_argmax_rows(const float* x, int64_t* out, int rows, int cols, cudaStream_t s) {
  const int wpb = kThreads / 32;
  int blocks = (rows + wpb - 1) / wpb;
  if (blocks > 132 * 8) blocks = 132 * 8;
  if (blocks < 1) blocks = 1;
  COLEARN_LAUNCH(argmax_rows_kernel, blocks, kThreads, 0, s, x, out, rows, cols);
  return cudaGetLastError();
}
cudaError_t launch_minmax_scale(const float* x, float* out, int rows, int cols, cudaStream_t s) {
  COLEARN_LAUNCH(minmax_scale_kernel, cols, 1024, 0, s, x, out, rows, cols);
  return cudaGetLastError();
}
cudaError_t launch_feistel_permutation(int* out, int n, int rows, uint64_t seed, cudaStream_t s) {
  COLEARN_LAUNCH(feistel_perm_kernel, grid_for((int64_t)n * rows, 1), kThreads, 0, s, out, n, rows, seed);
  return cudaGetLastError();
}
cudaError_t launch_fp32_to_bf16(const float* in, void* out, int64_t n, cudaStream_t s) {
  COLEARN_LAUNCH(fp32_to_bf16_kernel, grid_for(n), kThreads, 0, s, in, reinterpret_cast<__nv_bfloat16*>(out), n);
  return cudaGetLastError();
}
cudaError_t launch_transpose_bf16(const void* in, void* out, int rows, int cols, cudaStream_t s) {
  dim3 grid((cols + 31) / 32, (rows + 31) / 32), block(32, 8);
  COLEARN_LAUNCH(transpose_bf16_kernel, grid, block, 0, s, reinterpret_cast<const __nv_bfloat16*>(in), reinterpret_cast<__nv_bfloat16*>(out), rows, cols);
  return cudaGetLastError();
}
cudaError_t launch_fix_precision(const float* x, long long* out, int64_t n, double base, cudaStream_t s) {
  COLEARN_LAUNCH(fix_precision_kernel, grid_for(n, 1), kThreads, 0, s, x, out, n, base);
  return cudaGetLastError();
}
cudaError_t launch_float_precision(const long long* x, float* out, int64_t n, double inv_base, cudaStream_t s) {
  COLEARN_LAUNCH(float_precision_kernel, grid_for(n, 1), kThreads, 0, s, x, out, n, inv_base);
  return cudaGetLastError();
}
cudaError_t launch_ring_matmul(const long long* A, const long long* B, long long* C, int M, int K, int N, cudaStream_t s) {
  dim3 grid((N + 15) / 16, (M + 15) / 16), block(16, 16);
  COLEARN_LAUNCH(ring_matmul_kernel, grid, block, 0, s, reinterpret_cast<const unsigned long long*>(A),
                 reinterpret_cast<const unsigned long long*>(B), reinterpret_cast<unsigned long long*>(C), M, K, N);
  return cudaGetLastError();
}
cudaError_t launch_bias_sgd_from_partials(float* bias, const float* partials, int rows, int n, int64_t row_stride, float lr,
                                          float* grad_out, int n_bias, cudaStream_t s) {
  COLEARN_LAUNCH(bias_sgd_from_partials_kernel, (n + 255) / 256, 256, 0, s, bias, partials, rows, n, row_stride, lr, grad_out, n_bias);
  return cudaGetLastError();
}
cudaError_t launch_l2_flush(float* buf, int64_t n, cudaStream_t s) {
  COLEARN_LAUNCH(l2_flush_kernel, 132 * 8, kThreads, 0, s, buf, n);
  return cudaGetLastError();
}

}  // namespace colearn
