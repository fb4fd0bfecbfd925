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

#include <type_traits>

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

// Whether a row loader also names a second destination of the new theta (the version ring of ROWS_F32_BASED): the store of
// the step writes it in the same pass.  Off for every other loader.
template <class Rows>
struct RingWrite {
  static constexpr bool kOn = false;
  __device__ __forceinline__ static float* out(const Rows&) { return nullptr; }
};

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
    const float r = (opt.kind == SOPT_SGD) ? fmaf(opt.lr, a - t, t) : server_opt_step(opt, j, t, a);
    theta[j] = r;
    if constexpr (RingWrite<Slots>::kOn) RingWrite<Slots>::out(slots)[j] = r;
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
// optimizer step (OPT true); 16-byte accesses of theta and the moments per 4 elements inside n when vec.  RING: the new values
// are also stored to ring (16-byte stores when vec)
template <bool OPT, bool RING = false>
__device__ __forceinline__ void apply8(float* __restrict__ theta, int64_t e0, int64_t n, bool vec, const float (&acc)[8],
                                       const ServerOptArgs& opt, float* __restrict__ ring = nullptr) {
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
      if constexpr (RING) *reinterpret_cast<float4*>(ring + e) = t;
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (e + i < n) {
          const float t = theta[e + i], a = t + acc[4 * h + i];
          const float r = OPT ? server_opt_step(opt, e + i, t, a) : fmaf(opt.lr, a - t, t);
          theta[e + i] = r;
          if constexpr (RING) ring[e + i] = r;
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
// ROWS_F32_BASED: fp32 models trained from older global versions, each read as its delta to its own base, the ring slot
// base[k] (ring [slots][n]).  The loader of the robust body (stream / cached / average), of the distance passes (load8) and of
// fedavg_based_kernel; ring_out = ring + write_slot n receives the new theta.  vec: models, ring and n allow 16-byte loads.
struct BasedRows {
  static constexpr bool kDelta = true;
  const float* p;
  int64_t stride;
  const float* ring;
  const int* base;
  float* ring_out;
  int64_t n;
  bool vec;
  __device__ __forceinline__ const float* base_row(int k) const { return ring + (int64_t)__ldg(base + k) * n; }
  template <LdHint HINT>
  __device__ __forceinline__ void load8(int k, int64_t e0, float (&x)[8]) const {
    float b[8];
    lane_load8<HINT>(p + k * stride, e0, n, vec, x);
    lane_load8<kLdReadOnly>(base_row(k), e0, n, vec, b);   // a base is shared by every row trained from that version
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = x[i] - b[i];
  }
  __device__ __forceinline__ float stream(int c, int64_t j) const { return __ldcs(p + c * stride + j) - __ldg(base_row(c) + j); }
  __device__ __forceinline__ float cached(int c, int64_t j) const { return __ldg(p + c * stride + j) - __ldg(base_row(c) + j); }
  __device__ __forceinline__ float average(float a, float t) const { return t + a; }
};
template <>
struct RingWrite<BasedRows> {
  static constexpr bool kOn = true;
  __device__ __forceinline__ static float* out(const BasedRows& r) { return r.ring_out; }
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
__device__ __forceinline__ void dagg_dist_body(Rows rows, const float* __restrict__ theta, int k, DistAggScratch sc, int64_t n) {
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
template <class Rows>
__global__ void __launch_bounds__(kDaThreads)
dagg_dist_kernel(Rows rows, const float* __restrict__ theta, int k, DistAggScratch sc, int64_t n) {
  dagg_dist_body(rows, theta, k, sc, n);
}

// A geomed step l < L fused with the next distance pass: the lane forms c^l for its 8 elements from the current weights (c^0
// when no row is left), then the chunk sums of (x_k - c^l)^2, in one read of the rows.  KMAX > 0: k <= KMAX, the rows' 8 values
// stay in registers between the two loops; KMAX = 0: any k, the second loop rereads them through L1 / L2.
template <int KMAX, class Rows>
__device__ __forceinline__ void dagg_center_body(Rows rows, const float* __restrict__ theta, int k, DistAggScratch sc, int64_t n) {
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
template <int KMAX, class Rows>
__global__ void __launch_bounds__(kDaThreads, 1)
dagg_center_kernel(Rows rows, const float* __restrict__ theta, int k, DistAggScratch sc, int64_t n) {
  dagg_center_body<KMAX>(rows, theta, k, sc, n);
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
// (OPT true); 16-byte accesses of theta and the moments per 4 elements inside n when vec.  RING: the new values are also stored
// to ring
template <bool OPT, bool RING = false>
__device__ __forceinline__ void step_to8(float* __restrict__ theta, int64_t e0, int64_t n, bool vec, const float (&t)[8],
                                         const float (&a)[8], const ServerOptArgs& opt, float* __restrict__ ring = nullptr) {
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
      if constexpr (RING) *reinterpret_cast<float4*>(ring + e) = tt;
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (e + i < n) {
          const float tv = t[4 * h + i], av = a[4 * h + i];
          const float r = OPT ? server_opt_step(opt, e + i, tv, av) : fmaf(opt.lr, av - tv, tv);
          theta[e + i] = r;
          if constexpr (RING) ring[e + i] = r;
        }
      }
    }
  }
}

// Last pass: the aggregate from the final weights (geomed: c^L, or c^0 when no row is left; norm_clip: c^0 + the clipped sum),
// theta + it for deltas, and the server step on theta with the moments in place.
template <class Rows, bool CLIP, bool OPT>
__device__ __forceinline__ void dagg_apply_body(Rows rows, float* __restrict__ theta, int k, DistAggScratch sc, ServerOptArgs opt, int64_t n) {
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
    step_to8<OPT, RingWrite<Rows>::kOn>(theta, e0, n, vec, t, a, opt, RingWrite<Rows>::out(rows));
  }
}
template <class Rows, bool CLIP, bool OPT>
__global__ void __launch_bounds__(kDaThreads)
dagg_apply_kernel(Rows rows, float* __restrict__ theta, int k, DistAggScratch sc, ServerOptArgs opt, int64_t n) {
  dagg_apply_body<Rows, CLIP, OPT>(rows, theta, k, sc, opt, n);
}

// ---- asynchronous buffered aggregation (ROWS_F32_BASED) -------------------------------------------------------------------------
// The fp32 twin of fedavg_q_kernel on rows of mixed base versions: per element acc = fmaf(w_k, x_k - ring[base_k], acc) in slot
// order from +0, a = theta + acc, the step of apply8, and the new theta stored to theta and ring_out in the same pass.  One warp
// per 256 elements, lane l holding 8 of them.
template <bool OPT>
__global__ void __launch_bounds__(256)
fedavg_based_kernel(float* __restrict__ theta, BasedRows rows, const float* __restrict__ weights, int k, ServerOptArgs opt, int64_t n) {
  __shared__ float sw[StagedWeights::kSw];
  const StagedWeights staged(sw, weights, k);
  const int lane = threadIdx.x & 31;
  const int64_t nblk = uq_nblk(n);
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const bool vec = rows.vec && (((uintptr_t)theta | (uintptr_t)opt.m | (uintptr_t)opt.v) & 15) == 0;
  for (int64_t blk = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); blk < nblk; blk += warps) {
    const int64_t e0 = blk * kUqBlock + lane * 8;
    if (e0 >= n) continue;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll 2
    for (int c = 0; c < k; ++c) {
      const float w = staged.wt(c);
      float d[8];
      rows.load8<kLdStream>(c, e0, d);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(w, d[i], acc[i]);
    }
    apply8<OPT, true>(theta, e0, n, vec, acc, opt, rows.ring_out);
  }
}

// robust aggregate of the deltas to their bases: the body of fedavg_robust_kernel with the based loader (and its ring store)
template <int KMAX>
__global__ void __launch_bounds__(256)
fedavg_based_robust_kernel(float* __restrict__ theta, BasedRows rows, int k, AggArgs agg, ServerOptArgs opt, int64_t n) {
  fedavg_robust_body<KMAX>(theta, rows, k, agg, opt, n);
}

// the distance passes on based rows: the bodies of dagg_dist_kernel / dagg_center_kernel / dagg_apply_kernel under their own
// kernel names
__global__ void __launch_bounds__(kDaThreads)
dagg_based_dist_kernel(BasedRows rows, const float* __restrict__ theta, int k, DistAggScratch sc, int64_t n) {
  dagg_dist_body(rows, theta, k, sc, n);
}
template <int KMAX>
__global__ void __launch_bounds__(kDaThreads, 1)
dagg_based_center_kernel(BasedRows rows, const float* __restrict__ theta, int k, DistAggScratch sc, int64_t n) {
  dagg_center_body<KMAX>(rows, theta, k, sc, n);
}
template <bool CLIP, bool OPT>
__global__ void __launch_bounds__(kDaThreads)
dagg_based_apply_kernel(BasedRows rows, float* __restrict__ theta, int k, DistAggScratch sc, ServerOptArgs opt, int64_t n) {
  dagg_apply_body<BasedRows, CLIP, OPT>(rows, theta, k, sc, opt, n);
}
// the kernel of each distance pass for a row loader
template <class Rows> inline auto dagg_dist_for(const Rows&) { return dagg_dist_kernel<Rows>; }
inline auto dagg_dist_for(const BasedRows&) { return dagg_based_dist_kernel; }
template <int KMAX, class Rows> inline auto dagg_center_for(const Rows&) { return dagg_center_kernel<KMAX, Rows>; }
template <int KMAX> inline auto dagg_center_for(const BasedRows&) { return dagg_based_center_kernel<KMAX>; }
template <bool CLIP, bool OPT, class Rows> inline auto dagg_apply_for(const Rows&) { return dagg_apply_kernel<Rows, CLIP, OPT>; }
template <bool CLIP, bool OPT> inline auto dagg_apply_for(const BasedRows&) { return dagg_based_apply_kernel<CLIP, OPT>; }

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

// ---- detection-metrics summary (eval_summary.cuh) ---------------------------------------------------------------------------
// One CTA per (segment, chunk) work unit at a time, one thread per row (kEsRowsPerThread rows per thread and chunk).  The counts
// of the CTA's current segment accumulate in shared memory as uint32 and are flushed (non-zero words, 64-bit atomics) when the
// CTA moves to another segment and at the end.  A hot bin — a trained detector puts most rows into bin 0 or B - 1 — would take
// up to 32 shared atomics per warp on one word: the lanes with equal words are matched first and one leader adds the count.
__device__ __forceinline__ void es_count(unsigned* __restrict__ sm, int word) {
  const unsigned peers = __match_any_sync(0xffffffffu, word);
  if (word >= 0 && (int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(sm + word, (unsigned)__popc(peers));
}
__device__ __forceinline__ void es_flush(unsigned* __restrict__ sm, int64_t len, int64_t* __restrict__ dst) {
  __syncthreads();
  for (int64_t i = threadIdx.x; i < len; i += kEsThreads) {
    const unsigned v = sm[i];
    if (v != 0u) {
      atomicAdd(reinterpret_cast<unsigned long long*>(dst + i), (unsigned long long)v);
      sm[i] = 0u;
    }
  }
  __syncthreads();
}

// C = 1: the row's loss (0 for an invalid row), its confusion and histogram words (-1: none)
__device__ __forceinline__ double es_row_binary(const EvalSummaryArgs& a, int64_t row, bool in, int& conf, int& hist) {
  conf = hist = -1;
  if (!in) return 0.0;
  const float p = a.scores[row];
  const int y = es_label(a.labels[row], 1);
  if (!(p >= 0.f && p <= 1.f) || y < 0) return 0.0;            // (NaN fails the range test)
  conf = (int)es_conf_off() + 2 * y + (p > a.threshold ? 1 : 0);
  hist = (int)es_hist_off(1) + y * a.bins + es_bin(p, a.bins);
  return es_bce(p, y);
}

template <bool MULTI>
__global__ void __launch_bounds__(kEsThreads) eval_summary_kernel(const EvalSummaryArgs a) {
  constexpr int kEsFinalTile = 1024;
  COLEARN_DYN_SMEM(unsigned, sm);
  __shared__ double red[kEsThreads / 32];
  __shared__ double tile[kEsFinalTile];
  __shared__ int s_last;
  const int C = a.classes, B = a.bins, lane = threadIdx.x & 31;
  const int64_t L = es_row_len(C, B);
  const int64_t* offsets = a.table;
  const int64_t* unit_seg = a.table + a.segments + 1;
  const int64_t* seg_unit0 = unit_seg + a.units;
  int64_t* counts = a.out;
  double* loss = reinterpret_cast<double*>(a.out + (int64_t)a.segments * L);
  unsigned* ticket = reinterpret_cast<unsigned*>(a.out + (int64_t)a.segments * L + a.segments);
  double* partial = reinterpret_cast<double*>(a.out + (int64_t)a.segments * L + a.segments + 1);
  for (int64_t i = threadIdx.x; i < L; i += kEsThreads) sm[i] = 0u;
  int64_t cur = -1;
  __syncthreads();
  for (int64_t u = blockIdx.x; u < a.units; u += gridDim.x) {
    const int64_t s = unit_seg[u];
    if (s != cur) {
      if (cur >= 0) es_flush(sm, L, counts + cur * L);
      cur = s;
    }
    const int64_t r0 = offsets[s] + (u - seg_unit0[s]) * kEsChunk;
    const int64_t r1 = r0 + kEsChunk < offsets[s + 1] ? r0 + kEsChunk : offsets[s + 1];
    double acc = 0.0;
    if (!MULTI) {
      int conf[kEsRowsPerThread], hist[kEsRowsPerThread];
      double l[kEsRowsPerThread];
#pragma unroll
      for (int i = 0; i < kEsRowsPerThread; ++i) {
        const int64_t row = r0 + threadIdx.x + (int64_t)i * kEsThreads;
        l[i] = es_row_binary(a, row, row < r1, conf[i], hist[i]);
      }
      int bad = 0;
#pragma unroll
      for (int i = 0; i < kEsRowsPerThread; ++i) {
        acc += l[i];
        bad += (r0 + threadIdx.x + (int64_t)i * kEsThreads < r1 && conf[i] < 0) ? 1 : 0;
        es_count(sm, conf[i]);
        es_count(sm, hist[i]);
      }
      bad = __reduce_add_sync(0xffffffffu, bad);
      if (lane == 0 && bad != 0) atomicAdd(sm + 1, (unsigned)bad);
    } else {
      int bad = 0;
      for (int i = 0; i < kEsRowsPerThread; ++i) {
        const int64_t row = r0 + threadIdx.x + (int64_t)i * kEsThreads;
        const bool in = row < r1;
        const float* z = a.scores + row * C;
        // pass 1: finite, max, argmax (on finite scores argmax_takes is v > best: the lowest index among equals)
        int y = -1, arg = 0;
        float m = 0.f;
        if (in) {
          y = es_label(a.labels[row], C);
          bool finite = true;
          for (int c = 0; c < C; ++c) {
            const float v = z[c];
            finite = finite && isfinite(v);
            if (c == 0 || v > m) { m = v; arg = c; }
          }
          if (!finite) y = -1;
          bad += y < 0 ? 1 : 0;
        }
        // pass 2 (from L1): the float64 softmax denominator and the loss
        double sum = 0.0;
        if (y >= 0) {
          for (int c = 0; c < C; ++c) sum += exp((double)z[c] - (double)m);
          acc += log(sum) - ((double)z[y] - (double)m);
        }
        es_count(sm, y >= 0 ? (int)es_conf_off() + C * y + arg : -1);
        // pass 3 (from L1): the histogram of every class's softmax score
        for (int c = 0; c < C; ++c) {
          int word = -1;
          if (y >= 0) word = (int)es_hist_off(C) + (2 * c + (y == c ? 1 : 0)) * B + es_bin(exp((double)z[c] - (double)m) / sum, B);
          es_count(sm, word);
        }
      }
      bad = __reduce_add_sync(0xffffffffu, bad);
      if (lane == 0 && bad != 0) atomicAdd(sm + 1, (unsigned)bad);
    }
    acc = warp_tree_f64(acc);
    if (lane == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = red[0];
#pragma unroll
      for (int w = 1; w < kEsThreads / 32; ++w) t += red[w];
      partial[u] = t;
      sm[0] += (unsigned)(r1 - r0);
    }
    __syncthreads();
  }
  if (cur >= 0) es_flush(sm, L, counts + cur * L);
  // the last CTA adds every segment's chunk sums in chunk order
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(ticket, 1u) == gridDim.x - 1 ? 1 : 0;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // The partials come into shared memory a tile at a time, loaded by the whole CTA (one L2 round trip per chunk in the adding
  // thread would cost ~50 us at the full Bot-IoT set); a segment's running sum waits in loss[s] (zeroed by the launcher).
  for (int64_t base = 0; base < a.units; base += kEsFinalTile) {
    const int64_t n = a.units - base < kEsFinalTile ? a.units - base : kEsFinalTile;
    for (int64_t i = threadIdx.x; i < n; i += kEsThreads) tile[i] = __ldcg(partial + base + i);
    __syncthreads();
    for (int64_t s = threadIdx.x; s < a.segments; s += kEsThreads) {
      const int64_t lo = seg_unit0[s] > base ? seg_unit0[s] : base, hi = seg_unit0[s + 1] < base + n ? seg_unit0[s + 1] : base + n;
      if (lo >= hi) continue;
      double t = loss[s];
      for (int64_t u = lo; u < hi; ++u) t += tile[u - base];
      loss[s] = t;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *ticket = 0u;
}

// ---- reconstruction-error summary (recon_summary.cuh) -----------------------------------------------------------------------
// The work units, shared-memory counts (es_count / es_flush) and the chunk-order float64 sum of eval_summary_kernel; one thread
// per row computes the row's error over its D columns.
constexpr int kRsFinalTile = 1024;

// After every CTA flushed: the last CTA (by ticket) adds every segment's chunk sums in chunk order into sum[s] (zeroed by the
// launcher) and re-arms the ticket.  tile: kRsFinalTile doubles of shared memory.
__device__ __forceinline__ void rs_sum_chunks_in_order(const double* partial, unsigned* ticket, double* sum, const int64_t* seg_unit0,
                                                       int64_t segments, int64_t units, double* tile, int* s_last) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) *s_last = atomicAdd(ticket, 1u) == gridDim.x - 1 ? 1 : 0;
  __syncthreads();
  if (!*s_last) return;
  __threadfence();
  for (int64_t base = 0; base < units; base += kRsFinalTile) {
    const int64_t n = units - base < kRsFinalTile ? units - base : kRsFinalTile;
    for (int64_t i = threadIdx.x; i < n; i += kEsThreads) tile[i] = __ldcg(partial + base + i);
    __syncthreads();
    for (int64_t s = threadIdx.x; s < segments; s += kEsThreads) {
      const int64_t lo = seg_unit0[s] > base ? seg_unit0[s] : base, hi = seg_unit0[s + 1] < base + n ? seg_unit0[s + 1] : base + n;
      if (lo >= hi) continue;
      double t = sum[s];
      for (int64_t u = lo; u < hi; ++u) t += tile[u - base];
      sum[s] = t;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *ticket = 0u;
}

__global__ void __launch_bounds__(kEsThreads) recon_summary_kernel(const ReconSummaryArgs a) {
  COLEARN_DYN_SMEM(unsigned, sm);
  __shared__ double red[kEsThreads / 32];
  __shared__ double tile[kRsFinalTile];
  __shared__ int s_last;
  const int B = a.bins, D = a.dim, lane = threadIdx.x & 31, sub = rs_sub_log2(B);
  const int64_t L = rs_row_len(B);
  const int64_t* offsets = a.table;
  const int64_t* unit_seg = a.table + a.segments + 1;
  const int64_t* seg_unit0 = unit_seg + a.units;
  int64_t* counts = a.out;
  double* sum = reinterpret_cast<double*>(a.out + (int64_t)a.segments * L);
  unsigned* ticket = reinterpret_cast<unsigned*>(a.out + (int64_t)a.segments * L + a.segments);
  double* partial = reinterpret_cast<double*>(a.out + (int64_t)a.segments * L + a.segments + 1);
  for (int64_t i = threadIdx.x; i < L; i += kEsThreads) sm[i] = 0u;
  int64_t cur = -1;
  __syncthreads();
  for (int64_t u = blockIdx.x; u < a.units; u += gridDim.x) {
    const int64_t s = unit_seg[u];
    if (s != cur) {
      if (cur >= 0) es_flush(sm, L, counts + cur * L);
      cur = s;
    }
    const int64_t r0 = offsets[s] + (u - seg_unit0[s]) * kEsChunk;
    const int64_t r1 = r0 + kEsChunk < offsets[s + 1] ? r0 + kEsChunk : offsets[s + 1];
    double acc = 0.0;
    int bad = 0;
    for (int i = 0; i < kEsRowsPerThread; ++i) {
      const int64_t row = r0 + threadIdx.x + (int64_t)i * kEsThreads;
      int word = -1;
      if (row < r1) {
        const float* ph = a.xhat + row * D;
        const float* px = a.x + row * D;
        double e = 0.0;
        bool finite = true;
        for (int c = 0; c < D; ++c) {
          const float h = ph[c], v = px[c];
          finite = finite && isfinite(h) && isfinite(v);
          const double d = (double)(h - v);
          e += d * d;
        }
        int y = 0;
        if (a.labels != nullptr) {
          const float l = a.labels[row];
          y = l == 0.f ? 0 : (l == 1.f ? 1 : -1);
        }
        const bool valid = finite && y >= 0;
        const int b = rs_bin(e, sub);
        if (a.err != nullptr) a.err[row] = (float)e;
        if (a.flag != nullptr) a.flag[row] = (!valid || b >= a.alarm_bin) ? 1 : 0;
        if (valid) {
          acc += e;
          word = 2 + y * B + b;
        } else {
          ++bad;
        }
      }
      es_count(sm, word);
    }
    bad = __reduce_add_sync(0xffffffffu, bad);
    if (lane == 0 && bad != 0) atomicAdd(sm + 1, (unsigned)bad);
    acc = warp_tree_f64(acc);
    if (lane == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = red[0];
#pragma unroll
      for (int w = 1; w < kEsThreads / 32; ++w) t += red[w];
      partial[u] = t;
      sm[0] += (unsigned)(r1 - r0);
    }
    __syncthreads();
  }
  if (cur >= 0) es_flush(sm, L, counts + cur * L);
  rs_sum_chunks_in_order(partial, ticket, sum, seg_unit0, a.segments, a.units, tile, &s_last);
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

// local-optimizer step of a strided block (launch_local_opt_apply): one element per thread, grid-stride
__global__ void local_opt_apply_kernel(float* __restrict__ theta, int64_t ld, const float* __restrict__ grad, int64_t g_ld, int g_rows,
                                       float* __restrict__ m, float* __restrict__ v, int rows, int cols, LocalOptArgs a, LocalOptStep st,
                                       float lr) {
  const int64_t n = (int64_t)rows * cols, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t r = i / cols, c = i - r * cols;
    float g = 0.f;
    for (int p = 0; p < g_rows; ++p) g += grad[(r * g_rows + p) * g_ld + c];
    const int64_t e = r * ld + c;
    float mm = m != nullptr ? m[e] : 0.f, vv = v != nullptr ? v[e] : 0.f;
    local_opt_elem(a, st, lr, theta[e], g, mm, vv);
    if (m != nullptr) m[e] = mm;
    if (v != nullptr) v[e] = vv;
  }
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
namespace {
// The smallest register path that holds k: f(std::integral_constant<int, KMAX>) with KMAX 4, 8, 16, 32 (LARGEST 32) or 0, the
// general path.  A robust kind's register path costs KMAX^2 compares per element whatever k is; the geomed centre pass holds 8
// KMAX floats of rows per lane, so LARGEST 16 is the largest that stays clear of spills.
template <int LARGEST, class F>
inline void with_kmax(int k, F&& f) {
  if (k <= 4) f(std::integral_constant<int, 4>{});
  else if (k <= 8) f(std::integral_constant<int, 8>{});
  else if (k <= 16) f(std::integral_constant<int, 16>{});
  else if (LARGEST >= 32 && k <= 32) f(std::integral_constant<int, (LARGEST >= 32 ? 32 : 0)>{});
  else f(std::integral_constant<int, 0>{});
}
// The passes of one distance-based aggregation: the distance pass, its finalisation, then per geomed step l < L the fused centre
// + distance pass and its finalisation, and the apply pass: 2 L + 1 launches (norm_clip: 3).  grid <= 0: one CTA per chunk up to
// the persistent grid.
template <class Rows, bool CLIP, bool OPT>
inline void launch_dagg_apply_t(Rows rows, float* theta, int k, const DistAggScratch& sc, const ServerOptArgs& opt, int64_t n, int grid,
                                cudaStream_t s) {
  auto kernel = dagg_apply_for<CLIP, OPT>(rows);
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
    auto kernel = dagg_dist_for(rows);
    COLEARN_LAUNCH(kernel, grid, kDaThreads, 0, s, rows, theta, k, sc, n);
  }
  COLEARN_LAUNCH(dagg_finalize_kernel, k, kDaThreads, 0, s, sc, alpha, k, g, w_out, nchunks);
  const int steps = g.kind == DAGG_GEOMED ? g.iters - 1 : 0;
  for (int l = 0; l < steps; ++l) {
    with_kmax<16>(k, [&](auto kmax) {
      auto kernel = dagg_center_for<decltype(kmax)::value>(rows);
      COLEARN_LAUNCH(kernel, grid, kDaThreads, 0, s, rows, theta, k, sc, n);
    });
    COLEARN_LAUNCH(dagg_finalize_kernel, k, kDaThreads, 0, s, sc, alpha, k, g, w_out, nchunks);
  }
  const bool clip = g.kind == DAGG_NORM_CLIP, o = opt.kind != SOPT_SGD;
  if (clip && o) launch_dagg_apply_t<Rows, true, true>(rows, theta, k, sc, opt, n, grid, s);
  else if (clip) launch_dagg_apply_t<Rows, true, false>(rows, theta, k, sc, opt, n, grid, s);
  else if (o) launch_dagg_apply_t<Rows, false, true>(rows, theta, k, sc, opt, n, grid, s);
  else launch_dagg_apply_t<Rows, false, false>(rows, theta, k, sc, opt, n, grid, s);
  return cudaGetLastError();
}
}  // namespace

cudaError_t launch_topk_delta(const float* models, int64_t model_stride, const float* theta, float* residual, int64_t residual_stride,
                              int rows, int topk, uint8_t* indices, float* values, int64_t entries, int64_t n, cudaStream_t s) {
  if (rows < 1 || topk < 1 || topk > kUtMaxK || n < 1 || model_stride < n || residual_stride < n || entries < ut_entries(n, topk))
    return cudaErrorInvalidValue;
  COLEARN_LAUNCH(topk_delta_kernel, grid_for_warps(rows * uq_nblk(n)), kThreads, 0, s, models, model_stride, theta,
                 residual, residual_stride, rows, topk, indices, values, entries, n);
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
namespace {
inline bool is_distance_agg(int kind) { return kind == DAGG_GEOMED || kind == DAGG_NORM_CLIP; }
// the layout checks of each row format
inline bool rows_ok(const ClientRows& r, int64_t n) {
  switch (r.format) {
    case ROWS_F32: return r.stride >= n;
    case ROWS_INT8: return uq_layout_ok(8, r.payload, r.stride, n);
    case ROWS_INT4: return uq_layout_ok(4, r.payload, r.stride, n);
    case ROWS_TOPK: return r.topk >= 1 && r.topk <= kUtMaxK && n >= 1 && r.stride >= ut_entries(n, r.topk);
    case ROWS_SECAGG:
      return n >= 1 && n < kSaMaxElems && r.stride >= n && r.streams >= 0 && r.n_mean >= 1 && r.frac_bits >= 0 && r.frac_bits <= 64 &&
             (reinterpret_cast<uintptr_t>(r.keys) & 15) == 0;
    case ROWS_F32_BASED: {
      // the ring slot the step writes must not be a base of any row: the pass reads the bases while it stores the new theta
      if (r.stride < n || r.ring == nullptr || (reinterpret_cast<uintptr_t>(r.ring) & 15) != 0 || r.ring_slots < 2 ||
          r.write_slot < 0 || r.write_slot >= r.ring_slots || r.base_slot == nullptr || r.base_slot_host == nullptr)
        return false;
      for (int i = 0; i < r.k; ++i) {
        const int b = r.base_slot_host[i];
        if (b < 0 || b >= r.ring_slots || b == r.write_slot) return false;
      }
      return true;
    }
  }
  return false;
}
// Which aggregators a row format admits.  Top-k and secure-aggregation rows take only the mean: a coordinate-wise median of
// k/256-sparse deltas is 0 wherever fewer than half the rows kept the coordinate, their distances measure which entries the
// codec kept, and the masks leave the coordinator nothing but the sum.
inline bool agg_admissible(int format, int kind) {
  return kind == AGG_MEAN || format == ROWS_F32 || format == ROWS_INT8 || format == ROWS_INT4 || format == ROWS_F32_BASED;
}
inline cudaError_t route_based(float* theta, const ClientRows& r, const AggArgs& agg, const DistAggArgs& g, const ServerOptArgs& opt,
                               int64_t n, const ApplyWork& w, cudaStream_t s) {
  const bool vec = (((uintptr_t)r.models | (uintptr_t)r.ring) & 15) == 0 && (r.stride & 3) == 0 && (n & 3) == 0;
  const BasedRows rows{r.models, r.stride, r.ring, r.base_slot, r.ring + (int64_t)r.write_slot * n, n, vec};
  if (is_distance_agg(g.kind)) return launch_dagg_t(rows, theta, r.weights, r.k, g, opt, n, w.scratch, w.weights_out, w.grid, s);
  if (agg.kind != AGG_MEAN) {
    with_kmax<32>(r.k, [&](auto kmax) {
      auto kernel = fedavg_based_robust_kernel<decltype(kmax)::value>;
      COLEARN_LAUNCH(kernel, grid_for(n, 1), kThreads, 0, s, theta, rows, r.k, agg, opt, n);
    });
  } else if (opt.kind == SOPT_SGD) {
    COLEARN_LAUNCH(fedavg_based_kernel<false>, grid_for_warps(uq_nblk(n)), kThreads, 0, s, theta, rows, r.weights, r.k, opt, n);
  } else {
    COLEARN_LAUNCH(fedavg_based_kernel<true>, grid_for_warps(uq_nblk(n)), kThreads, 0, s, theta, rows, r.weights, r.k, opt, n);
  }
  return cudaGetLastError();
}

template <int BITS>
inline cudaError_t route_quantized(float* theta, const ClientRows& r, const AggArgs& agg, const DistAggArgs& g,
                                          const ServerOptArgs& opt, int64_t n, const ApplyWork& w, cudaStream_t s) {
  if (is_distance_agg(g.kind))
    return launch_dagg_t(QRows<BITS>{r.payload, r.stride, r.scales, uq_nblk(n), n}, theta, r.weights, r.k, g, opt, n, w.scratch,
                         w.weights_out, w.grid, s);
  if (agg.kind != AGG_MEAN) {
    with_kmax<32>(r.k, [&](auto kmax) {
      auto kernel = fedavg_q_robust_kernel<decltype(kmax)::value, BITS>;
      COLEARN_LAUNCH(kernel, grid_for(n, 1), kThreads, 0, s, theta, r.payload, r.stride, r.scales, r.k, agg, opt, n);
    });
  } else if (opt.kind == SOPT_SGD) {
    auto kernel = fedavg_q_kernel<BITS, false>;
    COLEARN_LAUNCH(kernel, grid_for_warps(uq_nblk(n)), kThreads, 0, s, theta, r.payload, r.stride, r.scales, r.weights, r.k, opt, n);
  } else {
    auto kernel = fedavg_q_kernel<BITS, true>;
    COLEARN_LAUNCH(kernel, grid_for_warps(uq_nblk(n)), kThreads, 0, s, theta, r.payload, r.stride, r.scales, r.weights, r.k, opt, n);
  }
  return cudaGetLastError();
}
inline cudaError_t route_secagg(float* theta, const ClientRows& r, const ServerOptArgs& opt, int64_t n, const ApplyWork& w,
                                       cudaStream_t s) {
  const int64_t cols = (n + kSaWords - 1) / kSaWords;
  const int per = sa_streams_per_task(n, r.streams);
  const uint32_t* partial = nullptr;
  if (per > 0) {
    uint32_t* workspace = static_cast<uint32_t*>(w.scratch);
    cudaError_t e = cudaMemsetAsync(workspace, 0, (size_t)n * sizeof(uint32_t), s);
    if (e != cudaSuccess) return e;
    COLEARN_LAUNCH(secagg_streams_kernel, grid_for(cols * ((r.streams + per - 1) / per), 1), kThreads, 0, s, r.keys, r.signs, r.streams,
                   per, workspace, n);
    partial = workspace;
  }
  const float inv_scale = ldexpf(1.f, -r.frac_bits), nf = (float)r.n_mean;
  if (opt.kind == SOPT_SGD) {
    COLEARN_LAUNCH(fedavg_secagg_kernel<false>, grid_for(cols, 1), kThreads, 0, s, theta, r.masked, r.stride, r.k, r.keys, r.signs,
                   r.streams, partial, inv_scale, nf, opt, n);
  } else {
    COLEARN_LAUNCH(fedavg_secagg_kernel<true>, grid_for(cols, 1), kThreads, 0, s, theta, r.masked, r.stride, r.k, r.keys, r.signs,
                   r.streams, partial, inv_scale, nf, opt, n);
  }
  return cudaGetLastError();
}
// The kernel instance of each (format, aggregator, optimizer) that launch_fedavg_apply admits.
inline cudaError_t route_fedavg_apply(float* theta, const ClientRows& r, const AggArgs& agg, const DistAggArgs& g,
                                      const ServerOptArgs& opt, int64_t n, const ApplyWork& w, cudaStream_t s) {
  switch (r.format) {
    case ROWS_F32:
      if (is_distance_agg(g.kind)) {
        const bool vec = ((uintptr_t)r.models & 15) == 0 && (r.stride & 3) == 0 && (n & 3) == 0;
        return launch_dagg_t(F32Rows{r.models, r.stride, n, vec}, theta, r.weights, r.k, g, opt, n, w.scratch, w.weights_out, w.grid, s);
      }
      if (agg.kind != AGG_MEAN) {
        with_kmax<32>(r.k, [&](auto kmax) {
          auto kernel = fedavg_robust_kernel<decltype(kmax)::value>;
          COLEARN_LAUNCH(kernel, grid_for(n, 1), kThreads, 0, s, theta, r.models, r.stride, r.k, agg, opt, n);
        });
      } else if (opt.kind == SOPT_SGD) {
        COLEARN_LAUNCH(fedavg_kernel<true>, grid_for(n), kThreads, 0, s, theta, r.models, r.stride, r.weights, r.k, opt.lr, n);
      } else {
        COLEARN_LAUNCH(fedavg_opt_kernel, grid_for(n), kThreads, 0, s, theta, r.models, r.stride, r.weights, r.k, opt, n);
      }
      return cudaGetLastError();
    case ROWS_INT8: return route_quantized<8>(theta, r, agg, g, opt, n, w, s);
    case ROWS_INT4: return route_quantized<4>(theta, r, agg, g, opt, n, w, s);
    case ROWS_TOPK:
      if (opt.kind == SOPT_SGD) {
        COLEARN_LAUNCH(fedavg_topk_kernel<false>, grid_for_warps(uq_nblk(n)), kThreads, 0, s, theta, r.indices, r.values, r.stride,
                       r.weights, r.k, r.topk, opt, n);
      } else {
        COLEARN_LAUNCH(fedavg_topk_kernel<true>, grid_for_warps(uq_nblk(n)), kThreads, 0, s, theta, r.indices, r.values, r.stride,
                       r.weights, r.k, r.topk, opt, n);
      }
      return cudaGetLastError();
    case ROWS_F32_BASED: return route_based(theta, r, agg, g, opt, n, w, s);
    default: return route_secagg(theta, r, opt, n, w, s);
  }
}
}  // namespace

size_t fedavg_apply_work_bytes(const ClientRows& rows, const AggregatorArgs& agg, int64_t n) {
  if (is_distance_agg(agg.kind) && agg_admissible(rows.format, agg.kind)) return (size_t)da_scratch_bytes(rows.k, n);
  if (rows.format == ROWS_SECAGG && sa_streams_per_task(n, rows.streams) > 0) return (size_t)n * sizeof(uint32_t);
  return 0;
}
cudaError_t launch_fedavg_apply(float* theta, const ClientRows& rows, const AggregatorArgs& a, const ServerOptArgs& opt, int64_t n,
                                const ApplyWork& work, cudaStream_t s) {
  const AggArgs agg{a.kind, a.trim};
  const DistAggArgs g{a.kind, a.iters, a.eps, a.clip};
  if (rows.k < 1 || !rows_ok(rows, n) || !server_opt_args_ok(opt) || !agg_admissible(rows.format, a.kind)) return cudaErrorInvalidValue;
  if (is_distance_agg(a.kind) ? n < 1 || !dist_agg_args_ok(g) : !agg_args_ok(agg)) return cudaErrorInvalidValue;
  if (fedavg_apply_work_bytes(rows, a, n) > 0 && (work.scratch == nullptr || (reinterpret_cast<uintptr_t>(work.scratch) & 15) != 0))
    return cudaErrorInvalidValue;
  return route_fedavg_apply(theta, rows, agg, g, opt, n, work, s);
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
cudaError_t launch_eval_summary(const EvalSummaryArgs& a, int grid, cudaStream_t s) {
  if (!eval_summary_args_ok(a.classes, a.bins, a.threshold) || a.segments < 1 || a.units < 0 ||
      (reinterpret_cast<uintptr_t>(a.out) & 7) != 0)
    return cudaErrorInvalidValue;
  const int64_t L = es_row_len(a.classes, a.bins);
  cudaError_t e = cudaMemsetAsync(a.out, 0, (size_t)((int64_t)a.segments * L + a.segments + 1) * sizeof(int64_t), s);
  if (e != cudaSuccess || a.units == 0) return e;
  const size_t smem = (size_t)L * sizeof(unsigned);
  auto kernel = a.classes == 1 ? eval_summary_kernel<false> : eval_summary_kernel<true>;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  if (grid <= 0) {
    int dev = 0, sms = 0;
    if ((e = cudaGetDevice(&dev)) != cudaSuccess || (e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess)
      return e;
    grid = (int)(a.units < 4 * sms ? a.units : 4 * sms);
  }
  COLEARN_LAUNCH(kernel, grid, kEsThreads, smem, s, a);
  return cudaGetLastError();
}
cudaError_t launch_recon_summary(const ReconSummaryArgs& a, int grid, cudaStream_t s) {
  if (!recon_summary_args_ok(a.dim, a.bins) || a.segments < 1 || a.units < 0 || (reinterpret_cast<uintptr_t>(a.out) & 7) != 0 ||
      (a.flag != nullptr && (a.alarm_bin < 0 || a.alarm_bin > a.bins)))
    return cudaErrorInvalidValue;
  const int64_t L = rs_row_len(a.bins);
  cudaError_t e = cudaMemsetAsync(a.out, 0, (size_t)((int64_t)a.segments * L + a.segments + 1) * sizeof(int64_t), s);
  if (e != cudaSuccess || a.units == 0) return e;
  const size_t smem = (size_t)L * sizeof(unsigned);
  e = cudaFuncSetAttribute(recon_summary_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  if (grid <= 0) {
    int dev = 0, sms = 0;
    if ((e = cudaGetDevice(&dev)) != cudaSuccess || (e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess)
      return e;
    grid = (int)(a.units < 4 * sms ? a.units : 4 * sms);
  }
  COLEARN_LAUNCH(recon_summary_kernel, grid, kEsThreads, smem, s, a);
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
cudaError_t launch_local_opt_apply(float* theta, int64_t ld, const float* grad, int64_t g_ld, int g_rows, float* m, float* v,
                                   int rows, int cols, LocalOptArgs a, LocalOptStep st, float lr, cudaStream_t s) {
  if (rows <= 0 || cols <= 0) return cudaSuccess;
  COLEARN_LAUNCH(local_opt_apply_kernel, grid_for((int64_t)rows * cols, 1), kThreads, 0, s, theta, ld, grad, g_ld, g_rows, m, v, rows,
                 cols, a, st, lr);
  return cudaGetLastError();
}
cudaError_t launch_l2_flush(float* buf, int64_t n, cudaStream_t s) {
  COLEARN_LAUNCH(l2_flush_kernel, 132 * 8, kThreads, 0, s, buf, n);
  return cudaGetLastError();
}

}  // namespace colearn
