// Cross-GPU collectives written directly against NVLink peer memory (no NCCL on these paths).
//
// The reference moves models with PySyft websocket RPC: train_config.send(worker)  (broadcast leg,
// client_federated.py:209), model_ptr.get() (gather leg, :211) and utils.federated_avg (CPU mean,
// federated_coordinator.py:373,568).  On an NVSwitch box every GPU maps every peer's symmetric
// arena, so those three legs become plain ld/st (or multimem.st) on peer addresses issued from
// inside the kernels that produce / consume the data:
//
//   star_round_kernel      (small models, latency-optimal, coordinator-centric)
//       wait(arrive flags) -> theta += lr_s * (sum_k slot_k - theta) -> st theta to every selected
//       peer inbox (P2P or NVLS multicast) -> last CTA raises the peers' bcast flags.
//       = FedAvg reduce + sample-count scale (pre-applied by producers) + server apply + next
//         round's broadcast in ONE kernel (SURVEY K1+K2+K3+K4).
//   twoshot_fedavg_kernel  (large models, bandwidth-optimal, symmetric)
//       rank r owns slice r: pulls w_k*theta_k[slice r] from every selected peer (P2P ld), applies
//       the server update, pushes the new slice into every peer's fp32 arena AND its bf16 shadow
//       (fp32->bf16 conversion fused into the broadcast), raising per-chunk ready flags that the
//       next round's first consumer GEMM polls from its TMA producer warp (fused broadcast->GEMM).
//   Both apply plain FedAvg with a server learning rate, or (template flag OPT) a FedOpt server optimizer step of
//   server_opt.cuh (FedAvgM / FedAdagrad / FedAdam / FedYogi) in the same pass.  With the template flag ROBUST the average
//   is the coordinate-wise median / trimmed mean of robust_agg.cuh instead of the weighted sum (unweighted, P2P only).
//
// Memory model: data stores are weak; a CTA finishes with __threadfence_system() and the flag is
// written with st.release.sys; consumers spin with ld.acquire.sys (and add fence.proxy.async before
// TMA reads — see gemm_tcgen05.cu).  Flags carry monotonically increasing epochs, never reset.
#include "colearn_kernels.h"
#include "produced.cuh"

#include <cuda_bf16.h>

#include <cstdio>
#ifdef COLEARN_HOST_SHIM
#include <stdlib.h>

#include <chrono>
#endif

namespace colearn {
namespace {

#ifdef COLEARN_HOST_SHIM
// CPU build (csrc/host_shim.h, tests): "peer" pointers are ordinary host pointers of the emulated ranks; the NVLS
// multimem forms have no host equivalent (the tests drive the P2P paths), release/acquire map to __atomic builtins
inline uint32_t ld_acquire_sys(const uint32_t* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
inline void st_release_sys(uint32_t* p, uint32_t v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
inline float4 ld_peer_f4(const float4* p) { return *p; }
inline void st_peer_f4(float4* p, const float4& v) { *p = v; }
inline void multimem_st_f4(float4*, const float4&) { abort(); }
inline float4 multimem_ld_reduce_f4(const float4*) { abort(); }
inline void multimem_st_b64(uint2*, const uint2&) { abort(); }
inline unsigned long long shim_globaltimer() {
  return (unsigned long long)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
inline uint32_t ld_acquire_gpu(const uint32_t* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
inline void st_release_gpu(uint32_t* p, uint32_t v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
#else
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ float4 ld_peer_f4(const float4* p) {
  // peer reads bypass L2 of the local GPU anyway; keep them out of L1 too (single use)
  float4 v;
  asm volatile("ld.global.relaxed.sys.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_peer_f4(float4* p, const float4& v) {
  asm volatile("st.global.relaxed.sys.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void multimem_st_f4(float4* p, const float4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 multimem_ld_reduce_f4(const float4* p) {
  // in-switch (NVLS) sum over every member of the multicast group: one 16-byte response per request
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void multimem_st_b64(uint2* p, const uint2& v) {
  asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)) : "memory");
}
__device__ __forceinline__ unsigned long long shim_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
#endif
__device__ __forceinline__ uint2 pack_bf16x4(const float4& v) {
  __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
  uint2 r;
  r.x = *reinterpret_cast<uint32_t*>(&a);
  r.y = *reinterpret_cast<uint32_t*>(&b);
  return r;
}

// -------------------------------------------------------------------------------------------------
// OPT = false: theta += server_lr (a - theta) (StarRoundArgs::opt.kind == 0); true: the server optimizer step of server_opt.cuh.
// ROBUST = false: a = sum of the (pre-weighted) slots; true: a = robust_agg.cuh over the raw slots of the arrived workers
template <bool OPT, bool ROBUST>
__global__ void __launch_bounds__(256)
star_round_kernel(StarRoundArgs a) {
  const int tid = threadIdx.x;
  // (1) wait for every selected worker's contribution of this round.  With a deadline (failure
  //     detection, SURVEY §5): block 0 decides who made it, publishes the arrived mask, and every block
  //     reduces over exactly that set, renormalising by the weight that actually arrived.
  uint32_t mask = a.select_mask;
  float renorm = 1.f;
  if (a.do_reduce) {
    if (a.timeout_ns == 0) {
      if (tid < a.world && ((mask >> tid) & 1u))
        spin_wait_ge(a.arrive_flags + tid, a.arrive_epoch, 20, "star_round: arrive flag of a selected worker");
      __syncthreads();
    } else {
      __shared__ uint32_t s_mask;
      if (blockIdx.x == 0) {
        if (tid == 0) s_mask = 0u;
        __syncthreads();
        if (tid < a.world && ((mask >> tid) & 1u)) {
          const unsigned long long t0 = shim_globaltimer();
          unsigned long long t1;
          bool ok = false;
          do {
            ok = ld_acquire_sys(a.arrive_flags + tid) >= a.arrive_epoch;
            t1 = shim_globaltimer();
          } while (!ok && (t1 - t0) < a.timeout_ns);
          if (ok) atomicOr(&s_mask, 1u << tid);
        }
        __syncthreads();
        if (tid == 0) {
          a.decision[1] = s_mask;
          __threadfence();
          st_release_gpu(a.decision, a.arrive_epoch);
        }
      } else {
        if (tid == 0) {
          uint32_t v;
          do { v = ld_acquire_gpu(a.decision); } while (v < a.arrive_epoch);
          s_mask = a.decision[1];
        }
      }
      __syncthreads();
      mask = s_mask;
      float wsum = 0.f, wall = 0.f;
      for (int k = 0; k < a.world; ++k) {
        if ((a.select_mask >> k) & 1u) wall += a.weights[k];
        if ((mask >> k) & 1u) wsum += a.weights[k];
      }
      renorm = wsum > 0.f ? wall / wsum : 0.f;
      if (mask == 0u) renorm = 0.f;
    }
  }
  const int64_t n4 = a.n >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  float4* theta4 = reinterpret_cast<float4*>(a.theta);
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + tid; j < n4; j += stride) {
    float4 t = theta4[j];
    if (a.do_reduce) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      if constexpr (ROBUST) {
        // the raw models of the arrived workers (slots k >= world do not exist), unweighted
        const uint32_t live = mask & ((1u << a.world) - 1u);
        const int n_live = __popc(live), b_trim = agg_trim_count(a.agg, n_live);
        float x[16], y[16], z[16], w[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if ((live >> k) & 1u) v = __ldcg(reinterpret_cast<const float4*>(a.slots + k * a.slot_stride) + j);
          x[k] = v.x; y[k] = v.y; z[k] = v.z; w[k] = v.w;
        }
        if (live == 0u) {
          acc = t;   // nobody arrived: keep theta
        } else {
          acc.x = agg_robust<16>(x, live, n_live, b_trim); acc.y = agg_robust<16>(y, live, n_live, b_trim);
          acc.z = agg_robust<16>(z, live, n_live, b_trim); acc.w = agg_robust<16>(w, live, n_live, b_trim);
        }
      } else {
        for (int k = 0; k < a.world; ++k) {
          if (!((mask >> k) & 1u)) continue;
          const float4 v = __ldcg(reinterpret_cast<const float4*>(a.slots + k * a.slot_stride) + j);
          acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        if (mask == 0u) acc = t;   // nobody arrived: keep theta
        else if (renorm != 1.f) { acc.x *= renorm; acc.y *= renorm; acc.z *= renorm; acc.w *= renorm; }
      }
      if constexpr (OPT) {
        if (mask != 0u) t = server_opt_step4(a.opt, j, t, acc);     // (nobody arrived: theta and the moments stay)
      } else {
        t.x = fmaf(a.server_lr, acc.x - t.x, t.x); t.y = fmaf(a.server_lr, acc.y - t.y, t.y);
        t.z = fmaf(a.server_lr, acc.z - t.z, t.z); t.w = fmaf(a.server_lr, acc.w - t.w, t.w);
      }
      theta4[j] = t;
    }
    if (a.do_bcast) {
      if (a.mc_inbox != nullptr) {
        multimem_st_f4(reinterpret_cast<float4*>(a.mc_inbox) + j, t);
      } else {
        for (int k = 0; k < a.world; ++k)
          if ((a.select_mask >> k) & 1u) st_peer_f4(reinterpret_cast<float4*>(a.peer_inbox[k]) + j, t);
      }
    }
  }
  // scalar tail (n not a multiple of 4)
  for (int64_t j = (n4 << 2) + (int64_t)blockIdx.x * blockDim.x + tid; j < a.n; j += stride) {
    float t = a.theta[j];
    if (a.do_reduce) {
      float acc = 0.f;
      if constexpr (ROBUST) {
        const uint32_t live = mask & ((1u << a.world) - 1u);
        const int n_live = __popc(live), b_trim = agg_trim_count(a.agg, n_live);
        float v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) v[k] = ((live >> k) & 1u) ? __ldcg(a.slots + k * a.slot_stride + j) : 0.f;
        acc = (live == 0u) ? t : agg_robust<16>(v, live, n_live, b_trim);
      } else {
        for (int k = 0; k < a.world; ++k)
          if ((mask >> k) & 1u) acc += __ldcg(a.slots + k * a.slot_stride + j);
        acc = (mask == 0u) ? t : acc * renorm;
      }
      if constexpr (OPT) {
        if (mask != 0u) t = server_opt_step(a.opt, j, t, acc);
      } else {
        t = fmaf(a.server_lr, acc - t, t);
      }
      a.theta[j] = t;
    }
    if (a.do_bcast)
      for (int k = 0; k < a.world; ++k)
        if ((a.select_mask >> k) & 1u) a.peer_inbox[k][j] = t;
  }
  // (3) last CTA publishes the broadcast epoch to every selected peer
  if (a.do_bcast) {
    __shared__ bool is_last;
    __threadfence_system();
    __syncthreads();
    if (tid == 0) {
      const unsigned prev = atomicAdd(a.grid_counter, 1u);
      is_last = (prev == gridDim.x - 1);
    }
    __syncthreads();
    if (is_last) {
      if (tid == 0) *a.grid_counter = 0u;
      __threadfence_system();
      if (tid < a.world && ((a.select_mask >> tid) & 1u)) st_release_sys(a.peer_bcast_flag[tid], a.bcast_epoch);
    }
  }
}

// robust_agg.cuh on each component of the float4 values v[k] of the ranks k in `valid` (the two-shot owner's registers; the
// other entries were never loaded and are not read)
__device__ __forceinline__ float4 agg_robust4(const float4 (&v)[8], uint32_t valid, int n, int b) {
  float x[8], y[8], z[8], w[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float4 u = ((valid >> k) & 1u) ? v[k] : make_float4(0.f, 0.f, 0.f, 0.f);
    x[k] = u.x; y[k] = u.y; z[k] = u.z; w[k] = u.w;
  }
  return make_float4(agg_robust<8>(x, valid, n, b), agg_robust<8>(y, valid, n, b), agg_robust<8>(z, valid, n, b),
                     agg_robust<8>(w, valid, n, b));
}

// -------------------------------------------------------------------------------------------------
// Two-shot FedAvg.  Work decomposition: the arena is cut into chunks of chunk_elems floats; chunk c
// belongs to rank (c % world) (interleaved ownership keeps every rank's NVLink ports busy for the
// whole kernel and lets early layers become ready first on every peer).  A CTA processes whole
// chunks so that it can publish the chunk's ready flag by itself.
// one owned chunk: pull it from every selected rank, apply, push it to every rank (fp32 + bf16), publish its flag.
// OPT: the server optimizer step (server_opt.cuh) on theta_prev with this rank's moment shards a.opt.m / a.opt.v, P2P path only.
// ROBUST: the median / trimmed mean of robust_agg.cuh over the ranks in `mask` instead of the weighted sum, P2P path only
template <bool OPT, bool ROBUST>
__device__ __forceinline__ void twoshot_chunk(const TwoShotArgs& a, const int64_t c, const float* sw, const int tid,
                                              const uint32_t mask, const bool use_mc) {
  const int64_t lo = c * a.chunk_elems;
  const int64_t hi = (lo + a.chunk_elems < a.n) ? lo + a.chunk_elems : a.n;
  const int64_t len4 = (hi - lo) >> 2;  // n and chunk_elems are multiples of 4
  if (use_mc) {
    // NVLS path (all ranks selected, uniform weights): the switch sums the W copies on the way in
    // (ingress P/W instead of (W-1)P/W) and replicates the result on the way out (egress P/W).
    const float w = sw[0];
    const float4* src = reinterpret_cast<const float4*>(a.mc_work) + (lo >> 2);
    float4* dst = reinterpret_cast<float4*>(a.mc_work) + (lo >> 2);
    uint2* dsh = a.mc_shadow ? reinterpret_cast<uint2*>(a.mc_shadow) + (lo >> 2) : nullptr;
    for (int64_t j = tid; j < len4; j += 4 * blockDim.x) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (j + u * blockDim.x < len4) v[u] = multimem_ld_reduce_f4(src + j + u * blockDim.x);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (j + u * blockDim.x < len4) {
          v[u].x *= w; v[u].y *= w; v[u].z *= w; v[u].w *= w;
          multimem_st_f4(dst + j + u * blockDim.x, v[u]);
          if (dsh) multimem_st_b64(dsh + j + u * blockDim.x, pack_bf16x4(v[u]));
          if (a.global_copy[0] != nullptr)
            for (int k = 0; k < a.world; ++k) st_peer_f4(reinterpret_cast<float4*>(a.global_copy[k]) + (lo >> 2) + j + u * blockDim.x, v[u]);
        }
      }
    }
  } else
  // two float4 per thread per iteration: 2 x (#selected peers) 16-byte peer loads in flight per thread
  for (int64_t j = tid; j < len4; j += 2 * blockDim.x) {
    const int64_t e4a = (lo >> 2) + j;
    const int64_t jb = j + blockDim.x;
    const bool has_b = jb < len4;
    const int64_t e4b = (lo >> 2) + jb;
    float4 va[8], vb[8];   // world <= 8 on an HGX box (checked by the launcher)
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (k < a.world && ((mask >> k) & 1u)) {
        va[k] = ld_peer_f4(reinterpret_cast<const float4*>(a.work[k]) + e4a);
        if (has_b) vb[k] = ld_peer_f4(reinterpret_cast<const float4*>(a.work[k]) + e4b);
      }
    }
    float4 acca = make_float4(0.f, 0.f, 0.f, 0.f), accb = make_float4(0.f, 0.f, 0.f, 0.f);
    if constexpr (ROBUST) {
      // the ranks that contribute, unweighted
      const uint32_t live = mask & ((1u << a.world) - 1u);
      const int n_live = __popc(live), b_trim = agg_trim_count(a.agg, n_live);
      acca = agg_robust4(va, live, n_live, b_trim);
      if (has_b) accb = agg_robust4(vb, live, n_live, b_trim);
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        if (k < a.world && ((mask >> k) & 1u)) {
          const float w = sw[k];
          acca.x = fmaf(w, va[k].x, acca.x); acca.y = fmaf(w, va[k].y, acca.y);
          acca.z = fmaf(w, va[k].z, acca.z); acca.w = fmaf(w, va[k].w, acca.w);
          if (has_b) {
            accb.x = fmaf(w, vb[k].x, accb.x); accb.y = fmaf(w, vb[k].y, accb.y);
            accb.z = fmaf(w, vb[k].z, accb.z); accb.w = fmaf(w, vb[k].w, accb.w);
          }
        }
      }
    }
    if constexpr (OPT) {
      // theta_prev is required with an optimizer (launch_twoshot_fedavg); the owner keeps the moments of its chunks
      float4 t = reinterpret_cast<float4*>(a.theta_prev)[e4a];
      t = server_opt_step4(a.opt, e4a, t, acca);
      reinterpret_cast<float4*>(a.theta_prev)[e4a] = t;
      acca = t;
      if (has_b) {
        float4 u = reinterpret_cast<float4*>(a.theta_prev)[e4b];
        u = server_opt_step4(a.opt, e4b, u, accb);
        reinterpret_cast<float4*>(a.theta_prev)[e4b] = u;
        accb = u;
      }
    } else if (a.theta_prev != nullptr) {
      float4 t = reinterpret_cast<float4*>(a.theta_prev)[e4a];
      t.x = fmaf(a.server_lr, acca.x - t.x, t.x); t.y = fmaf(a.server_lr, acca.y - t.y, t.y);
      t.z = fmaf(a.server_lr, acca.z - t.z, t.z); t.w = fmaf(a.server_lr, acca.w - t.w, t.w);
      reinterpret_cast<float4*>(a.theta_prev)[e4a] = t;
      acca = t;
      if (has_b) {
        float4 u = reinterpret_cast<float4*>(a.theta_prev)[e4b];
        u.x = fmaf(a.server_lr, accb.x - u.x, u.x); u.y = fmaf(a.server_lr, accb.y - u.y, u.y);
        u.z = fmaf(a.server_lr, accb.z - u.z, u.z); u.w = fmaf(a.server_lr, accb.w - u.w, u.w);
        reinterpret_cast<float4*>(a.theta_prev)[e4b] = u;
        accb = u;
      }
    }
    const uint2 pa = pack_bf16x4(acca), pb = pack_bf16x4(accb);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (k < a.world) {
        st_peer_f4(reinterpret_cast<float4*>(a.work[k]) + e4a, acca);
        if (a.shadow_bf16[k] != nullptr) reinterpret_cast<uint2*>(a.shadow_bf16[k])[e4a] = pa;
        if (a.global_copy[k] != nullptr) st_peer_f4(reinterpret_cast<float4*>(a.global_copy[k]) + e4a, acca);
        if (has_b) {
          st_peer_f4(reinterpret_cast<float4*>(a.work[k]) + e4b, accb);
          if (a.shadow_bf16[k] != nullptr) reinterpret_cast<uint2*>(a.shadow_bf16[k])[e4b] = pb;
          if (a.global_copy[k] != nullptr) st_peer_f4(reinterpret_cast<float4*>(a.global_copy[k]) + e4b, accb);
        }
      }
    }
  }
  __threadfence_system();
  __syncthreads();
  if (tid < a.world) {
    __threadfence_system();
    st_release_sys(a.chunk_flags[tid] + c, a.epoch);
  }
  __syncthreads();
}

// ROBUST instances run 256-thread CTAs (launch_twoshot_fedavg): the rank count over the owner's 2 x 8 float4 registers does
// not fit the 128 registers a 512-thread CTA leaves a thread without spilling
template <bool OPT, bool ROBUST>
__global__ void __launch_bounds__(ROBUST ? 256 : 512)
twoshot_fedavg_kernel(TwoShotArgs a) {
  const int tid = threadIdx.x;
  __shared__ float sw[16];
  __shared__ uint32_t s_mask;
  // (0) announce "my local training of this round is done" to every rank (stream order guarantees it is)
  if (a.signal_arrive && blockIdx.x == 0 && tid < a.world) {
    __threadfence_system();
    st_release_sys(a.peer_arrive[tid], a.epoch);
  }
  uint32_t mask = a.select_mask;
  if (a.deadline_ns == 0) {
    if (tid < a.world) {
      sw[tid] = a.weights[tid];
      if ((mask >> tid) & 1u) spin_wait_ge(a.arrive_flags + tid, a.epoch, 20, "twoshot_fedavg: arrive flag of a selected rank");
    }
    __syncthreads();
  } else {
    // failure detection: the coordinator (rank 0) decides who made it and tells everybody; every CTA of every rank then works on
    // the same arrived set
    const int slot = (int)(a.epoch & 7u);
    if (a.rank == 0 && blockIdx.x == 0) {
      if (tid == 0) s_mask = 0u;
      __syncthreads();
      if (tid < a.world && ((mask >> tid) & 1u)) {
        const unsigned long long t0 = shim_globaltimer();
        bool ok = false;
        do {
          ok = ld_acquire_sys(a.arrive_flags + tid) >= a.epoch;
        } while (!ok && (shim_globaltimer() - t0) < a.deadline_ns);
        if (ok) atomicOr(&s_mask, 1u << tid);
      }
      __syncthreads();
      if (tid < a.world) {
        a.decision[tid][2 * slot + 1] = s_mask;
        __threadfence_system();
        st_release_sys(a.decision[tid] + 2 * slot, a.epoch);
      }
      __syncthreads();
    }
    if (tid == 0) {
      spin_wait_ge(a.decision[a.rank] + 2 * slot, a.epoch, 20, "twoshot_fedavg: the coordinator's arrived-set decision of this round");
      // (a ring slot that already carries a LATER epoch: this rank is more than 8 rounds behind — it takes part in nothing)
      s_mask = (ld_acquire_sys(a.decision[a.rank] + 2 * slot) == a.epoch) ? a.decision[a.rank][2 * slot + 1] : 0u;
    }
    __syncthreads();
    mask = s_mask;
    if (tid < a.world) {
      float wsum = 0.f, wall = 0.f;
      for (int k = 0; k < a.world; ++k) {
        if ((a.select_mask >> k) & 1u) wall += a.true_weights[k];
        if ((mask >> k) & 1u) wsum += a.true_weights[k];
      }
      sw[tid] = (wsum > 0.f) ? a.true_weights[tid] * (wall / wsum) : 0.f;
    }
    __syncthreads();
  }
  const int64_t n_chunks = (a.n + a.chunk_elems - 1) / a.chunk_elems;
  // chunk ownership is dealt among the ranks that take part: the j-th of them owns chunks j, j + n_own, ...  (without a deadline
  // every rank of the box takes part, selected or not: owner of chunk c = c % world)
  const uint32_t full = (a.world >= 32) ? 0xffffffffu : ((1u << a.world) - 1u);
  const uint32_t owners = (a.deadline_ns != 0 && mask != 0u) ? mask : full;
  const int n_own = __popc(owners);
  const bool i_own = (owners >> a.rank) & 1u;
  const int my_idx = __popc(owners & ((1u << a.rank) - 1u));
  const bool use_mc = !OPT && !ROBUST && a.mc_work != nullptr && (a.deadline_ns == 0 || mask == full);
  if (i_own && mask != 0u) {
    for (int64_t oc = blockIdx.x; ; oc += gridDim.x) {
      const int64_t c = my_idx + oc * n_own;
      if (c >= n_chunks) break;
      twoshot_chunk<OPT, ROBUST>(a, c, sw, tid, mask, use_mc);
    }
  } else if (mask == 0u && a.rank == 0) {
    // nobody arrived in time: the model stays as it is; the coordinator still publishes the chunk flags so that nobody waits
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + tid; c < n_chunks; c += (int64_t)gridDim.x * blockDim.x)
      for (int k = 0; k < a.world; ++k) st_release_sys(a.chunk_flags[k] + c, a.epoch);
  }
  // (3) optionally hold the stream until the whole arena of THIS rank has been refreshed by its owners
  if (a.wait_all) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + tid; c < n_chunks; c += (int64_t)gridDim.x * blockDim.x)
      spin_wait_ge(a.chunk_flags[a.rank] + c, a.epoch, 40, "twoshot_fedavg: chunk flag of my arena (its owner never pushed it)");
  }
}

// deadline mode: a rank that missed the previous round's deadline restores its arena from the copy the owners pushed
__global__ void __launch_bounds__(512)
twoshot_resync_kernel(const uint32_t* ring, uint32_t prev_epoch, int rank, float* work, __nv_bfloat16* shadow, const float* global_copy, int64_t n) {
  const int slot = (int)(prev_epoch & 7u);
  const bool decided = ring[2 * slot] == prev_epoch;
  const bool was_in = decided && ((ring[2 * slot + 1] >> rank) & 1u);
  if (was_in || prev_epoch == 0u) return;
  const int64_t n4 = n >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n4; j += stride) {
    const float4 v = reinterpret_cast<const float4*>(global_copy)[j];
    reinterpret_cast<float4*>(work)[j] = v;
    if (shadow != nullptr) reinterpret_cast<uint2*>(shadow)[j] = pack_bf16x4(v);
  }
}

// Overlapped form (fused wgrad GEMM -> FedAvg reduce, produced.cuh): runs on a few CTAs NEXT TO the last local step.
// Chunks are taken in whatever order the producers of all selected ranks finish them (the backward pass finalises the
// last layers first): each CTA sweeps its owned chunks, newest-first, and processes those whose produced epochs have
// arrived from every selected rank.
template <bool OPT, bool ROBUST>
__global__ void __launch_bounds__(ROBUST ? 256 : 512)
twoshot_overlap_kernel(TwoShotArgs a) {
  const int tid = threadIdx.x;
  __shared__ float sw[16];
  __shared__ int s_ready;
  __shared__ unsigned long long s_done[8];      // up to 512 owned chunks per CTA and pass
  if (tid < a.world) sw[tid] = a.weights[tid];
  const int64_t n_chunks = (a.n + a.chunk_elems - 1) / a.chunk_elems;
  const int64_t owned = (n_chunks - a.rank + a.world - 1) / a.world;                  // c = rank + oc * world, oc < owned
  const int64_t mine = (owned - (int64_t)blockIdx.x + gridDim.x - 1) / gridDim.x;   // oc = blockIdx.x + i * gridDim.x, i < mine
  const unsigned long long t0 = shim_globaltimer();
  for (int64_t base = 0; base < mine; base += 512) {
    const int cnt = (int)((mine - base < 512) ? mine - base : 512);
    if (tid < 8) s_done[tid] = 0ull;
    __syncthreads();
    int left = cnt;
    while (left > 0) {
      int progressed = 0;
      for (int i = cnt - 1; i >= 0; --i) {
        if ((s_done[i >> 6] >> (i & 63)) & 1ull) continue;                         // uniform: read by all threads
        const int64_t c = a.rank + ((int64_t)blockIdx.x + (base + i) * gridDim.x) * a.world;
        if (tid == 0) s_ready = 1;
        __syncthreads();
        if (tid < a.world && ((a.select_mask >> tid) & 1u) && ld_acquire_sys(a.produced + (int64_t)tid * n_chunks + c) < a.epoch) s_ready = 0;
        __syncthreads();
        const int ready = s_ready;
        __syncthreads();
        if (!ready) continue;
        twoshot_chunk<OPT, ROBUST>(a, c, sw, tid, a.select_mask, !OPT && !ROBUST && a.mc_work != nullptr);
        if (tid == 0) s_done[i >> 6] |= 1ull << (i & 63);
        __syncthreads();
        --left;
        progressed = 1;
      }
      if (!progressed) {
        if (a.produced_timeout_ns != 0 && shim_globaltimer() - t0 > a.produced_timeout_ns) {
#ifndef COLEARN_HOST_SHIM
          if (tid == 0) printf("twoshot_overlap_kernel: rank %d block %d still waits for %d chunk(s) after %llu ns\n", a.rank, (int)blockIdx.x, left, a.produced_timeout_ns);
          __trap();
#else
          abort();
#endif
        }
        __nanosleep(200);
      }
    }
    __syncthreads();
  }
  if (a.wait_all) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + tid; c < n_chunks; c += (int64_t)gridDim.x * blockDim.x)
      spin_wait_ge(a.chunk_flags[a.rank] + c, a.epoch, 40, "twoshot_fedavg: chunk flag of my arena (its owner never pushed it)");
  }
}

// every element of [lo, hi) is final: one thread per chunk reports the overlap (kernel boundary = the stores are done)
__global__ void produced_mark_kernel(const ProducedSignal* sig, int64_t lo, int64_t hi) {
  const int64_t c = (lo >> sig->chunk_shift) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t c_lo = c << sig->chunk_shift, c_hi = (c + 1) << sig->chunk_shift;
  const int64_t b = lo > c_lo ? lo : c_lo, e = hi < c_hi ? hi : c_hi;
  if (e > b) {
    __threadfence_system();
    produced_add(sig, c, (uint32_t)(e - b));
  }
}

// Many clients per GPU: sum the C locally trained (already weight-scaled) client models and push the
// result into the coordinator's slot on a peer GPU, then raise this rank's arrive flag (last CTA).
__global__ void __launch_bounds__(256)
reduce_push_kernel(const float* __restrict__ slots, int k, int64_t stride, int64_t n, float* __restrict__ dst,
                   const float* __restrict__ losses, float* __restrict__ loss_dst, uint32_t* flag, uint32_t value,
                   uint32_t* counter) {
  const int64_t n4 = n >> 2;
  const int64_t gstride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n4; j += gstride) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int c = 0; c < k; ++c) {
      const float4 v = __ldcg(reinterpret_cast<const float4*>(slots + c * stride) + j);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    st_peer_f4(reinterpret_cast<float4*>(dst) + j, acc);
  }
  for (int64_t j = (n4 << 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gstride) {
    float acc = 0.f;
    for (int c = 0; c < k; ++c) acc += __ldcg(slots + c * stride + j);
    dst[j] = acc;
  }
  __shared__ bool is_last;
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (is_last && threadIdx.x == 0) {
    *counter = 0u;
    if (loss_dst != nullptr && losses != nullptr) {  // mean of the clients' {last, mean} losses
      float l0 = 0.f, l1 = 0.f;
      for (int c = 0; c < k; ++c) { l0 += __ldcg(losses + 2 * c); l1 += __ldcg(losses + 2 * c + 1); }
      loss_dst[0] = l0 / k;
      loss_dst[1] = l1 / k;
    }
    __threadfence_system();
    if (flag != nullptr) st_release_sys(flag, value);
  }
}

__global__ void set_flag_kernel(uint32_t* flag, uint32_t value) {
  __threadfence_system();
  st_release_sys(flag, value);
}
__global__ void signal_peers_kernel(PeerFlags f, int world, uint32_t value) {
  __threadfence_system();
  if ((int)threadIdx.x < world) st_release_sys(f.ptr[threadIdx.x], value);
}
__global__ void wait_flag_kernel(const uint32_t* flag, uint32_t value) {
  spin_wait_ge(flag, value, 50, "wait_flag");
}
// wait until every one of `count` consecutive flags reached `value`
__global__ void wait_flags_kernel(const uint32_t* flags, int count, uint32_t value) {
  for (int i = threadIdx.x; i < count; i += blockDim.x)
    spin_wait_ge(flags + i, value, 50, "wait_flags: chunk flag of the previous round's broadcast");
}

__global__ void wait_flags_dev_kernel(const uint32_t* flags, int count, const uint32_t* value_ptr) {
  const uint32_t value = ld_acquire_sys(value_ptr);
  for (int i = threadIdx.x; i < count; i += blockDim.x)
    spin_wait_ge(flags + i, value, 50, "wait_flags: chunk flag of the previous round's broadcast");
}

__global__ void __launch_bounds__(512)
p2p_copy_kernel(float* __restrict__ dst, const float* __restrict__ src, int64_t n, uint32_t* flag,
                uint32_t flag_value, uint32_t* counter) {
  const int64_t n4 = n >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int64_t j = i0; j < n4; j += stride) {
    const float4 v = ld_peer_f4(reinterpret_cast<const float4*>(src) + j);
    st_peer_f4(reinterpret_cast<float4*>(dst) + j, v);
  }
  for (int64_t j = (n4 << 2) + i0; j < n; j += stride) dst[j] = src[j];
  if (flag != nullptr) {
    __shared__ bool is_last;
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) is_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
    __syncthreads();
    if (is_last && threadIdx.x == 0) {
      *counter = 0u;
      __threadfence_system();
      st_release_sys(flag, flag_value);
    }
  }
}

}  // namespace

// (the plain FedAvg instances are referenced last: the cubin then lists them first for each kernel)
cudaError_t launch_star_round(const StarRoundArgs& a, int n_blocks, cudaStream_t s) {
  if (a.world > 16 || !server_opt_args_ok(a.opt) || !agg_args_ok(a.agg)) return cudaErrorInvalidValue;
  if (n_blocks < 1) n_blocks = 1;
  const bool opt = a.opt.kind != SOPT_SGD, robust = a.agg.kind != AGG_MEAN;
  if (robust && opt) {
    COLEARN_LAUNCH((star_round_kernel<true, true>), n_blocks, 256, 0, s, a);
  } else if (robust) {
    COLEARN_LAUNCH((star_round_kernel<false, true>), n_blocks, 256, 0, s, a);
  } else if (opt) {
    COLEARN_LAUNCH((star_round_kernel<true, false>), n_blocks, 256, 0, s, a);
  } else {
    COLEARN_LAUNCH((star_round_kernel<false, false>), n_blocks, 256, 0, s, a);
  }
  return cudaGetLastError();
}

cudaError_t launch_twoshot_fedavg(const TwoShotArgs& a, int n_blocks, cudaStream_t s) {
  if (a.world > 8 || (a.n & 3) || (a.chunk_elems & 3)) return cudaErrorInvalidValue;
  if (n_blocks < 1) n_blocks = 1;
  const bool opt = a.opt.kind != SOPT_SGD, robust = a.agg.kind != AGG_MEAN;
  if (opt) {
    // the moments are sharded by the fixed ownership c % world: no deadline (ownership follows the arrived set), no NVLS
    if (!server_opt_args_ok(a.opt) || a.theta_prev == nullptr || a.deadline_ns != 0 || a.mc_work != nullptr) return cudaErrorInvalidValue;
  }
  // robust: the switch of the NVLS path can only sum; a deadline is fine (a robust aggregate keeps no per-rank state)
  if (robust && (!agg_args_ok(a.agg) || a.mc_work != nullptr)) return cudaErrorInvalidValue;
  const bool overlap = a.produced != nullptr;
  if (robust && opt) {
    if (overlap) COLEARN_LAUNCH((twoshot_overlap_kernel<true, true>), n_blocks, 256, 0, s, a);
    else COLEARN_LAUNCH((twoshot_fedavg_kernel<true, true>), n_blocks, 256, 0, s, a);
  } else if (robust) {
    if (overlap) COLEARN_LAUNCH((twoshot_overlap_kernel<false, true>), n_blocks, 256, 0, s, a);
    else COLEARN_LAUNCH((twoshot_fedavg_kernel<false, true>), n_blocks, 256, 0, s, a);
  } else if (opt) {
    if (overlap) COLEARN_LAUNCH((twoshot_overlap_kernel<true, false>), n_blocks, 512, 0, s, a);
    else COLEARN_LAUNCH((twoshot_fedavg_kernel<true, false>), n_blocks, 512, 0, s, a);
  } else {
    if (overlap) COLEARN_LAUNCH((twoshot_overlap_kernel<false, false>), n_blocks, 512, 0, s, a);
    else COLEARN_LAUNCH((twoshot_fedavg_kernel<false, false>), n_blocks, 512, 0, s, a);
  }
  return cudaGetLastError();
}

cudaError_t launch_twoshot_resync(const uint32_t* decision_ring, uint32_t prev_epoch, int rank, float* work, void* shadow_bf16,
                                  const float* global_copy, int64_t n, int n_blocks, cudaStream_t s) {
  if (decision_ring == nullptr || work == nullptr || global_copy == nullptr || (n & 3)) return cudaErrorInvalidValue;
  COLEARN_LAUNCH(twoshot_resync_kernel, n_blocks < 1 ? 1 : n_blocks, 512, 0, s, decision_ring, prev_epoch, rank, work,
                 reinterpret_cast<__nv_bfloat16*>(shadow_bf16), global_copy, n);
  return cudaGetLastError();
}

cudaError_t launch_produced_mark(const ProducedSignal* sig_dev, int chunk_shift, int64_t lo, int64_t hi, cudaStream_t s) {
  if (sig_dev == nullptr || lo < 0 || hi < lo || chunk_shift < 2 || chunk_shift > 30) return cudaErrorInvalidValue;
  if (hi == lo) return cudaSuccess;
  const int64_t chunks = ((hi - 1) >> chunk_shift) - (lo >> chunk_shift) + 1;
  const int threads = 128;
  COLEARN_LAUNCH(produced_mark_kernel, (int)((chunks + threads - 1) / threads), threads, 0, s, sig_dev, lo, hi);
  return cudaGetLastError();
}

cudaError_t launch_signal_peers(const PeerFlags& flags, int world, uint32_t value, cudaStream_t s) {
  if (world > 16) return cudaErrorInvalidValue;
  COLEARN_LAUNCH(signal_peers_kernel, 1, 32, 0, s, flags, world, value);
  return cudaGetLastError();
}

cudaError_t launch_reduce_push(const float* slots, int k, int64_t stride, int64_t n, float* dst, const float* losses,
                               float* loss_dst, uint32_t* flag, uint32_t value, uint32_t* counter, int n_blocks,
                               cudaStream_t s) {
  if (n_blocks < 1) n_blocks = 1;
  COLEARN_LAUNCH(reduce_push_kernel, n_blocks, 256, 0, s, slots, k, stride, n, dst, losses, loss_dst, flag, value, counter);
  return cudaGetLastError();
}
cudaError_t launch_set_flag(uint32_t* flag, uint32_t value, cudaStream_t s) {
  COLEARN_LAUNCH(set_flag_kernel, 1, 1, 0, s, flag, value);
  return cudaGetLastError();
}
cudaError_t launch_wait_flag(const uint32_t* flag, uint32_t value, cudaStream_t s) {
  COLEARN_LAUNCH(wait_flag_kernel, 1, 1, 0, s, flag, value);
  return cudaGetLastError();
}
cudaError_t launch_wait_flags(const uint32_t* flags, int count, uint32_t value, cudaStream_t s) {
  COLEARN_LAUNCH(wait_flags_kernel, 1, 128, 0, s, flags, count, value);
  return cudaGetLastError();
}
cudaError_t launch_wait_flags_dev(const uint32_t* flags, int count, const uint32_t* value_ptr, cudaStream_t s) {
  COLEARN_LAUNCH(wait_flags_dev_kernel, 1, 128, 0, s, flags, count, value_ptr);
  return cudaGetLastError();
}
cudaError_t launch_p2p_copy(float* dst, const float* src, int64_t n, uint32_t* flag, uint32_t flag_value,
                            int n_blocks, cudaStream_t s) {
  static uint32_t* counter = nullptr;
  if (flag != nullptr && counter == nullptr) {
#ifdef COLEARN_HOST_SHIM
    counter = new uint32_t(0);
#else
    cudaError_t e = cudaMalloc(&counter, sizeof(uint32_t));
    if (e != cudaSuccess) return e;
    cudaMemset(counter, 0, sizeof(uint32_t));
#endif
  }
  if (n_blocks < 1) n_blocks = 1;
  COLEARN_LAUNCH(p2p_copy_kernel, n_blocks, 512, 0, s, dst, src, n, flag, flag_value, counter);
  return cudaGetLastError();
}

COLEARN_DEFINE_SPIN_LIMIT_SETTER(set_spin_limit_comm)

// CUDA loads a kernel's code lazily at its first launch, and that load can need the device to be idle.  Kernels of this file
// spin on flags that OTHER kernels raise (the overlapped two-shot waits for the last backward pass' reports; the workers wait
// for the coordinator's broadcast), so a kernel that is launched for the first time while a spinning kernel is resident can
// deadlock the device (e.g. the first produced_mark_kernel next to twoshot_overlap_kernel).  Touching the function
// attributes forces the load; the engine calls this once per device before any round.
cudaError_t preload_comm_kernels() {
#ifndef COLEARN_HOST_SHIM
  cudaFuncAttributes attr;
  const void* kernels[] = {(const void*)star_round_kernel<false, false>, (const void*)star_round_kernel<true, false>,
                           (const void*)star_round_kernel<false, true>, (const void*)star_round_kernel<true, true>,
                           (const void*)twoshot_fedavg_kernel<false, false>, (const void*)twoshot_fedavg_kernel<true, false>,
                           (const void*)twoshot_fedavg_kernel<false, true>, (const void*)twoshot_fedavg_kernel<true, true>,
                           (const void*)twoshot_overlap_kernel<false, false>, (const void*)twoshot_overlap_kernel<true, false>,
                           (const void*)twoshot_overlap_kernel<false, true>, (const void*)twoshot_overlap_kernel<true, true>,
                           (const void*)produced_mark_kernel, (const void*)twoshot_resync_kernel, (const void*)reduce_push_kernel, (const void*)set_flag_kernel,
                           (const void*)signal_peers_kernel, (const void*)wait_flag_kernel, (const void*)wait_flags_kernel,
                           (const void*)wait_flags_dev_kernel, (const void*)p2p_copy_kernel};
  for (const void* k : kernels) {
    cudaError_t e = cudaFuncGetAttributes(&attr, k);
    if (e != cudaSuccess) return e;
  }
#endif
  return cudaSuccess;
}

}  // namespace colearn
