// mlp_local_sgd_persistent — one launch = one worker's whole local fit.
//
// What it replaces: the worker-side loop of the reference (PySyft FederatedClient._fit, SURVEY
// C27, triggered at client_federated.py:210): for every batch { zero_grad; forward; loss;
// backward; SGD step } — ~15 tiny ATen kernels per step, 1000-3000 dependent steps per round.
//
// Design: the networks in play (FFNN 10-50-30-10-1, MLP 10-64-64-2, TestingRemote
// 2-50-10-1) have <= 5k parameters, so the *entire model lives in shared memory* for the whole
// fit and one CTA walks the dependent SGD steps with no global-memory traffic other than the
// streamed samples.  Batch-1 sequential SGD is inherently serial (SURVEY §7.3-2): tensor cores
// are irrelevant at these shapes; what matters is the per-step dependency chain, so
//   * every layer is spread over the CTA as (neuron, T-lane group) with a shuffle reduce,
//   * weight rows are padded so forward reads are bank-conflict free (stride == T mod 32),
//   * the same (neuron, lane) owns a weight in forward and in the update, so no barrier is
//     needed between a step's update and the next step's forward,
//   * activations are double buffered by step parity (removes one more barrier),
//   * samples are gathered through the permutation one chunk ahead into registers.
// One CTA = one federated client; gridDim.x clients train concurrently (VirtualWorker mode runs
// all K workers of a round in ONE launch).  The epilogue applies the client's FedAvg weight and
// writes w_k*theta_k (or the scaled delta) straight to theta_out — typically the coordinator's
// slot buffer on a peer GPU over NVLink — then raises a release flag (SURVEY K2/K4).
#include "colearn_kernels.h"

#include <math.h>
#include <type_traits>

namespace colearn {
namespace {

constexpr int NT = 256;      // threads per CTA
constexpr int CHUNK = 64;    // samples gathered per pipeline stage

// ---- compile-time network description ---------------------------------------------------------
template <int I, int D0, int... Rest>
struct DimAt { static constexpr int v = DimAt<I - 1, Rest...>::v; };
template <int D0, int... Rest>
struct DimAt<0, D0, Rest...> { static constexpr int v = D0; };

__host__ __device__ constexpr int pow2_floor(int x) { int p = 1; while (p * 2 <= x) p *= 2; return p; }
__host__ __device__ constexpr int group_size(int n_out, int k_in) {
  int t = pow2_floor(NT / n_out);
  if (t > 32) t = 32;
  while (t > 1 && t > k_in) t /= 2;
  return t;
}
__host__ __device__ constexpr int padded_stride(int k, int t) {
  int s = k;
  while ((s % 32) != (t % 32)) ++s;
  return s;
}

template <bool SIGMOID_OUT, int... Ds>
struct Net {
  static constexpr int L = sizeof...(Ds) - 1;
  static constexpr bool kSigmoid = SIGMOID_OUT;
  template <int I> static constexpr int dim() { return DimAt<I, Ds...>::v; }
  static constexpr int DIN = DimAt<0, Ds...>::v;
  static constexpr int DOUT = DimAt<L, Ds...>::v;
};

template <class N, int LI>
struct Layer {
  static constexpr int K = N::template dim<LI>();
  static constexpr int NO = N::template dim<LI + 1>();
  static constexpr int T = group_size(NO, K);        // lanes per output neuron (fwd/update)
  static constexpr int KP = padded_stride(K, T);     // padded smem row stride
  static constexpr int TB = group_size(K, NO);       // lanes per input neuron (dgrad)
  static constexpr int SMEM = NO * KP + NO;          // padded W + bias
  static constexpr int FLAT = NO * K + NO;           // unpadded arena footprint
};
template <class N, int LI> struct Offs {
  static constexpr int smem = Offs<N, LI - 1>::smem + Layer<N, LI - 1>::SMEM;
  static constexpr int flat = Offs<N, LI - 1>::flat + Layer<N, LI - 1>::FLAT;
  static constexpr int act = Offs<N, LI - 1>::act + N::template dim<LI>();   // a_{LI+1} offset
};
template <class N> struct Offs<N, 0> { static constexpr int smem = 0, flat = 0, act = 0; };
template <class N> struct Totals {
  static constexpr int smem_params = Offs<N, N::L>::smem;
  static constexpr int flat_params = Offs<N, N::L>::flat;
  static constexpr int acts = Offs<N, N::L>::act;      // sum of D1..DL (a_1..a_L)
  static constexpr int ROW_MAX = N::DIN + N::DOUT;     // x row + widest possible y row
  static constexpr int EPT = (CHUNK * ROW_MAX + NT - 1) / NT;
};

// ---- memory-model helpers ----------------------------------------------------------------------
#ifdef COLEARN_HOST_SHIM
inline uint32_t ld_acquire_sys(const uint32_t* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
inline void st_release_sys(uint32_t* p, uint32_t v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
#else
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
#endif

// max that keeps NaN, like torch.relu / torch.clamp: fmaxf(NaN, 0) is 0, which let a NaN sample train the rest of the model
// on zeros and report a finite loss.  max.NaN.f32 is still one FMNMX; without a NaN operand it gives the bits of fmaxf.
#ifdef COLEARN_HOST_SHIM
inline float fmax_nan(float a, float b) { return a != a ? a : (b != b ? b : fmaxf(a, b)); }
#else
__device__ __forceinline__ float fmax_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
#endif
__device__ __forceinline__ float relu_nan(float z) { return fmax_nan(z, 0.f); }
// ReLU backward as threshold_backward computes it: the gradient passes unless the activation is <= 0, so a NaN activation
// passes it on (`a > 0 ? g : 0` would zero it)
__device__ __forceinline__ float relu_grad(float a, float g) { return a <= 0.f ? 0.f : g; }

// ---- per-layer device functions ----------------------------------------------------------------
// OWN_ONLY (the training kernel): threads past the last (neuron, lane) pair skip the weight reads instead of shadowing
// the last neuron's row — their result was always discarded, but in the training loop those reads raced with the owner
// thread's rank-1 update of that row from the previous step (no barrier separates the two by design: every weight is read
// and written by the same thread).  Found by the CPU race check (scripts/racecheck_cpu.sh); the inference kernel keeps
// the original form.
template <class N, int LI, bool RELU, bool OWN_ONLY = false>
__device__ __forceinline__ void fwd_layer(const float* __restrict__ sP, const float* __restrict__ a_in,
                                          float* __restrict__ a_out, int tid) {
  using Ly = Layer<N, LI>;
  constexpr int K = Ly::K, NO = Ly::NO, T = Ly::T, KP = Ly::KP;
  const bool valid = tid < NO * T;
  const int n = valid ? tid / T : NO - 1;
  const int t = tid % T;
  const float* w = sP + Offs<N, LI>::smem + n * KP;
  float acc0 = 0.f, acc1 = 0.f;
  if (!OWN_ONLY || valid) {
#pragma unroll
    for (int k = t, j = 0; k < K; k += T, ++j) {
      if (j & 1) acc1 = fmaf(w[k], a_in[k], acc1);
      else acc0 = fmaf(w[k], a_in[k], acc0);
    }
  }
  float acc = acc0 + acc1;
#pragma unroll
  for (int o = T / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (valid && t == 0) {
    const float z = acc + sP[Offs<N, LI>::smem + NO * KP + n];
    a_out[n] = RELU ? relu_nan(z) : z;
  }
}

// dz_in[k] = relu'(a_in[k]) * sum_n W[n][k] * dz_out[n]
template <class N, int LI>
__device__ __forceinline__ void bwd_dh(const float* __restrict__ sP, const float* __restrict__ dz_out,
                                       const float* __restrict__ a_in, float* __restrict__ dz_in, int tid) {
  using Ly = Layer<N, LI>;
  constexpr int K = Ly::K, NO = Ly::NO, TB = Ly::TB, KP = Ly::KP;
  const bool valid = tid < K * TB;
  const int k = valid ? tid / TB : K - 1;
  const int t = tid % TB;
  const float* w = sP + Offs<N, LI>::smem + k;
  float acc0 = 0.f, acc1 = 0.f;
#pragma unroll
  for (int n = t, j = 0; n < NO; n += TB, ++j) {
    if (j & 1) acc1 = fmaf(w[n * KP], dz_out[n], acc1);
    else acc0 = fmaf(w[n * KP], dz_out[n], acc0);
  }
  float acc = acc0 + acc1;
#pragma unroll
  for (int o = TB / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (valid && t == 0) dz_in[k] = relu_grad(a_in[k], acc);
}

// P[n][k] += scale * dz_out[n] * a_in[k];  bias[n] += scale * dz_out[n]
template <class N, int LI>
__device__ __forceinline__ void rank1_update(float* __restrict__ sP, const float* __restrict__ dz_out,
                                             const float* __restrict__ a_in, float scale, int tid) {
  using Ly = Layer<N, LI>;
  constexpr int K = Ly::K, NO = Ly::NO, T = Ly::T, KP = Ly::KP;
  if (tid < NO * T) {
    const int n = tid / T, t = tid % T;
    const float g = scale * dz_out[n];
    float* w = sP + Offs<N, LI>::smem + n * KP;
#pragma unroll
    for (int k = t; k < K; k += T) w[k] = fmaf(g, a_in[k], w[k]);
    if (t == 0) sP[Offs<N, LI>::smem + NO * KP + n] += g;
  }
}

template <class N, int LI, bool OWN_ONLY = false>
struct FwdChain {
  static __device__ __forceinline__ void run(const float* sP, const float* a0, float* acts, int tid) {
    constexpr bool last = (LI == N::L - 1);
    const float* a_in = (LI == 0) ? a0 : acts + Offs<N, LI - (LI > 0)>::act;
    float* a_out = acts + Offs<N, LI>::act;
    fwd_layer<N, LI, !last, OWN_ONLY>(sP, a_in, a_out, tid);
    __syncthreads();
    if constexpr (!last) FwdChain<N, LI + 1, OWN_ONLY>::run(sP, a0, acts, tid);
  }
};

template <class N, int LI>
struct BwdChain {
  // dzs holds dz_1..dz_L at the same offsets as a_1..a_L.
  static __device__ __forceinline__ void run(float* sP, float* sTarget, const float* a0,
                                             const float* acts, float* dzs, float scale, int tid) {
    const float* a_in = (LI == 0) ? a0 : acts + Offs<N, LI - (LI > 0)>::act;
    const float* dz_out = dzs + Offs<N, LI>::act;
    if constexpr (LI > 0) {
      bwd_dh<N, LI>(sP, dz_out, a_in, dzs + Offs<N, LI - 1>::act, tid);
      __syncthreads();  // all reads of W_LI done before it is updated; dz_{LI} visible
    }
    rank1_update<N, LI>(sTarget, dz_out, a_in, scale, tid);
    if constexpr (LI > 0) BwdChain<N, LI - 1>::run(sP, sTarget, a0, acts, dzs, scale, tid);
  }
};

// Loss + gradient w.r.t. the last pre-activation, computed by warp 0 (DOUT <= 32).
template <class N>
__device__ __forceinline__ float loss_and_dz(float* aL, float* dzL, const float* yrow, int loss,
                                             float inv_b, int lane) {
  constexpr int DO = N::DOUT;
  float value = 0.f;
  if (loss == LOSS_XENT) {
    const float z = lane < DO ? aL[lane] : -INFINITY;
    float m = z;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    const float e = lane < DO ? __expf(z - m) : 0.f;
    float s = e;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const int label = (int)yrow[0];
    const float zl = __shfl_sync(0xffffffffu, z, label & 31);
    value = (__logf(s) + m) - zl;
    if (lane < DO) dzL[lane] = (e / s - (lane == label ? 1.f : 0.f)) * inv_b;
  } else {
    float contrib = 0.f;
    if (lane < DO) {
      const float z = aL[lane];
      const float y = yrow[lane];
      float out = z, dact = 1.f;
      if (N::kSigmoid) { out = 1.f / (1.f + __expf(-z)); dact = out * (1.f - out); aL[lane] = out; }
      if (loss == LOSS_BCE) {
        const float lp = fmax_nan(__logf(out), -100.f), l1p = fmax_nan(log1pf(-out), -100.f);
        contrib = -(y * lp + (1.f - y) * l1p) * (1.f / DO);
        dzL[lane] = (out - y) * inv_b * (1.f / DO);
      } else {  // SSE / MSE
        const float d = out - y;
        contrib = d * d;
        dzL[lane] = 2.f * d * dact * ((loss == LOSS_MSE) ? inv_b : 1.f);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, o);
    value = contrib;
  }
  return value;
}

// Arena <-> padded smem (recursion over layers; everything is compile-time)
template <class N, int LI>
struct ParamIO {
  using Ly = Layer<N, LI>;
  static constexpr int K = Ly::K, NO = Ly::NO, KP = Ly::KP;
  static constexpr int SO = Offs<N, LI>::smem, FO = Offs<N, LI>::flat;
  template <bool CG>
  static __device__ __forceinline__ float ld(const float* p) { return CG ? __ldcg(p) : __ldg(p); }

  template <bool CG>
  static __device__ __forceinline__ void load(float* __restrict__ sP, const float* __restrict__ theta, int tid) {
    for (int i = tid; i < NO * KP; i += NT) {
      const int n = i / KP, k = i - n * KP;
      sP[SO + i] = (k < K) ? ld<CG>(theta + FO + n * K + k) : 0.f;
    }
    for (int i = tid; i < NO; i += NT) sP[SO + NO * KP + i] = ld<CG>(theta + FO + NO * K + i);
    if constexpr (LI + 1 < N::L) ParamIO<N, LI + 1>::template load<CG>(sP, theta, tid);
  }
  static __device__ __forceinline__ void store(const float* __restrict__ sP, const float* __restrict__ theta_in,
                                               float* __restrict__ theta_out, float w, int delta_mode, int tid) {
    for (int i = tid; i < NO * K; i += NT) {
      const int n = i / K, k = i - n * K;
      float v = sP[SO + n * KP + k];
      if (delta_mode) v -= __ldcg(theta_in + FO + i);
      theta_out[FO + i] = w * v;
    }
    for (int i = tid; i < NO; i += NT) {
      float v = sP[SO + NO * KP + i];
      if (delta_mode) v -= __ldcg(theta_in + FO + NO * K + i);
      theta_out[FO + NO * K + i] = w * v;
    }
    if constexpr (LI + 1 < N::L) ParamIO<N, LI + 1>::store(sP, theta_in, theta_out, w, delta_mode, tid);
  }
};

// ---- the kernel ----------------------------------------------------------------------------------
template <class N>
__global__ void __launch_bounds__(NT, 1)
mlp_local_sgd_kernel(const ClientDesc* __restrict__ descs, SgdHyper hp) {
  using Tot = Totals<N>;
  constexpr int SP = Tot::smem_params;
  constexpr int DIN = N::DIN, DOUT = N::DOUT, ROWM = Tot::ROW_MAX, EPT = Tot::EPT;
  COLEARN_DYN_SMEM(float, smem);

  const ClientDesc d = descs[blockIdx.x];
  const int tid = threadIdx.x;
  const int B = hp.batch_size < 1 ? 1 : hp.batch_size;
  const bool accumulate = B > 1;

  float* sP = smem;                              // padded params
  float* sG = sP + SP;                           // gradient accumulator (only touched if B > 1)
  float* sAct = sG + (accumulate ? SP : 0);      // 2 x acts (double buffered by step parity)
  float* sDz = sAct + 2 * Tot::acts;             // dz_1..dz_L
  float* sData = sDz + Tot::acts;                // 2 x CHUNK x ROWM sample ring
  float* sMisc = sData + 2 * CHUNK * ROWM;       // [0] last loss, [1] loss sum

  // (1) wait for the broadcast of this round's global model to land (SURVEY K1/K4)
  if (d.wait_flag != nullptr) {
    if (tid == 0) {
      spin_wait_ge(d.wait_flag, d.wait_value, 32, "mlp_local_sgd: broadcast flag of this round");
    }
    __syncthreads();
  }

  // (2) global arena -> padded smem layout (L1 bypass: the arena may be peer-written)
  ParamIO<N, 0>::template load<true>(sP, d.theta_in, tid);
  if (accumulate)
    for (int i = tid; i < SP; i += NT) sG[i] = 0.f;
  if (tid < 2) sMisc[tid] = 0.f;

  // (3) step bookkeeping
  const int n = d.n;
  const int ydim = d.y_dim;
  const int row = DIN + ydim;
  const int spe = ((n > 0 ? n : 1) + B - 1) / B;  // steps per epoch (an empty shard: Q = 0 below, see the v2 kernel)
  long long total_steps = (long long)hp.epochs * spe;
  if (hp.max_steps > 0 && hp.max_steps < total_steps) total_steps = hp.max_steps;
  // total samples consumed by those steps
  long long Q;
  {
    const long long full_epochs = total_steps / spe;
    const long long rem_steps = total_steps - full_epochs * spe;
    long long rem_samples = rem_steps * B;
    if (rem_samples > n) rem_samples = n;
    Q = full_epochs * (long long)n + rem_samples;
  }
  const int n_chunks = (int)((Q + CHUNK - 1) / CHUNK);

  const FeistelDomain fdom = feistel_domain((uint32_t)(n > 0 ? n : 1));   // in-kernel shuffle (ClientDesc::perm_seed)
  float pre[EPT];
  auto issue_loads = [&](int chunk) {
#pragma unroll
    for (int j = 0; j < EPT; ++j) {
      const int e = tid + j * NT;
      pre[j] = 0.f;
      if (e < CHUNK * row) {
        const int i = e / row, c = e - i * row;
        const long long q = (long long)chunk * CHUNK + i;
        if (q < Q) {
          const int ep = (int)(q / n);
          const int pos = (int)(q - (long long)ep * n);
          const int idx = d.perm ? __ldg(d.perm + (size_t)(ep % d.perm_rows) * n + pos)
                                 : (d.perm_seed ? (int)feistel_index((uint32_t)pos, (uint32_t)n, fdom, d.perm_seed, d.perm_row0 + ep) : pos);
          pre[j] = (c < DIN) ? __ldg(d.x + (size_t)idx * DIN + c) : __ldg(d.y + (size_t)idx * ydim + (c - DIN));
        }
      }
    }
  };
  auto store_loads = [&](int buf) {
    float* dst = sData + buf * (CHUNK * ROWM);
#pragma unroll
    for (int j = 0; j < EPT; ++j) {
      const int e = tid + j * NT;
      if (e < CHUNK * row) dst[e] = pre[j];
    }
  };

  if (n_chunks > 0) { issue_loads(0); store_loads(0); }
  __syncthreads();

  long long step = 0;
  int pos_in_epoch = 0;   // samples consumed in the current epoch
  int in_batch = 0;       // samples accumulated in the current batch
  int cur_batch = (n < B) ? n : B;
  float batch_loss = 0.f;  // only meaningful on tid 0
  int parity = 0;

  for (int c = 0; c < n_chunks; ++c) {
    if (c + 1 < n_chunks) issue_loads(c + 1);  // next chunk's gathers fly during this chunk's math
    const float* chunk = sData + (c & 1) * (CHUNK * ROWM);
    const long long q0 = (long long)c * CHUNK;
    const int cnt = (int)((Q - q0) < CHUNK ? (Q - q0) : CHUNK);
    for (int i = 0; i < cnt; ++i) {
      const float* a0 = chunk + i * row;
      const float* yrow = a0 + DIN;
      float* acts = sAct + parity * Tot::acts;
      const float inv_b = 1.f / (float)cur_batch;

      FwdChain<N, 0, true>::run(sP, a0, acts, tid);
      if (tid < 32) {
        const float v = loss_and_dz<N>(acts + Offs<N, N::L - 1>::act, sDz + Offs<N, N::L - 1>::act,
                                       yrow, hp.loss, inv_b, tid);
        if (tid == 0) batch_loss += (hp.loss == LOSS_SSE) ? v : v * inv_b;
      }
      __syncthreads();
      BwdChain<N, N::L - 1>::run(sP, accumulate ? sG : sP, a0, acts, sDz,
                                 accumulate ? 1.f : -hp.lr, tid);
      parity ^= 1;

      ++in_batch;
      ++pos_in_epoch;
      if (in_batch == cur_batch) {  // batch closes -> SGD step
        if (accumulate) {
          __syncthreads();
          for (int k = tid; k < SP; k += NT) { sP[k] = fmaf(-hp.lr, sG[k], sP[k]); sG[k] = 0.f; }
          __syncthreads();
        }
        if (tid == 0) { sMisc[0] = batch_loss; sMisc[1] += batch_loss; batch_loss = 0.f; }
        ++step;
        in_batch = 0;
        if (pos_in_epoch >= n) pos_in_epoch = 0;
        const int left = n - pos_in_epoch;
        cur_batch = left < B ? left : B;
      }
    }
    __syncthreads();                 // everyone is done reading chunk buffers of this parity
    if (c + 1 < n_chunks) store_loads((c + 1) & 1);
    __syncthreads();
  }
  __syncthreads();

  // (4) epilogue: out_scale * theta_k (or scaled delta) -> theta_out (possibly a peer GPU)
  ParamIO<N, 0>::store(sP, d.theta_in, d.theta_out, d.out_scale, d.delta_mode, tid);
  if (tid == 0 && d.loss_out != nullptr) {
    d.loss_out[0] = sMisc[0];
    d.loss_out[1] = step > 0 ? sMisc[1] / (float)step : 0.f;
  }
  __syncthreads();
  if (tid == 0 && d.signal_flag != nullptr) {
    __threadfence_system();
    st_release_sys(d.signal_flag, d.signal_value);
  }
}


// =====================================================================================================
// v2: register-resident weights.
//
// v1 keeps the weights in shared memory, so its step waits on shared-memory weight reads / read-modify-write updates
// and on barriers.  v2 removes shared
// memory from the weight path entirely: every thread keeps, in registers and for the whole fit,
//   wr[KC]  its slice of row n of W_l       (forward + update, (neuron n, lane t) mapping)
//   wt[NC]  its slice of column k of W_l    (dgrad,            (input  k, lane t') mapping)
// Both copies receive the *same* fmaf sequence (dz[n] * a[k]) so they never diverge, the update is a
// pure register FFMA, the barrier between dgrad and update disappears (weights are thread-private)
// and only activations / dz vectors travel through shared memory.  128 threads = one warp per SMSP.
// =====================================================================================================
#define V2_NS v2_128
#define V2_NT 128
#include "mlp_v2.cuh"
#undef V2_NS
#undef V2_NT
// 128 threads, blocked reduction slices + pre-scaled dz (see the V2_BLOCKED comment in mlp_v2.cuh)
#define V2_NS v2_128b
#define V2_NT 128
#define V2_BLOCKED 1
#include "mlp_v2.cuh"
#undef V2_BLOCKED
#undef V2_NS
#undef V2_NT
// the blocked kernel with its FMAs written in pairs (see the V2_PACKED comment in mlp_v2.cuh)
#define V2_NS v2_128p
#define V2_NT 128
#define V2_BLOCKED 1
#define V2_PACKED 1
#include "mlp_v2.cuh"
#undef V2_PACKED
#undef V2_BLOCKED
#undef V2_NS
#undef V2_NT

// ---- batched forward (inference / evaluation) --------------------------------------------------------
template <class N>
__global__ void __launch_bounds__(NT, 1)
mlp_forward_kernel(const float* __restrict__ theta, const float* __restrict__ x, float* __restrict__ out, int n) {
  using Tot = Totals<N>;
  constexpr int SP = Tot::smem_params;
  constexpr int L = N::L, DIN = N::DIN, DOUT = N::DOUT;
  COLEARN_DYN_SMEM(float, smem);
  float* sP = smem;
  float* sX = sP + SP;
  float* sAct = sX + DIN;
  const int tid = threadIdx.x;
  ParamIO<N, 0>::template load<false>(sP, theta, tid);
  __syncthreads();
  for (int s = blockIdx.x; s < n; s += gridDim.x) {
    if (tid < DIN) sX[tid] = x[(size_t)s * DIN + tid];
    __syncthreads();
    FwdChain<N, 0>::run(sP, sX, sAct, tid);
    if (tid < DOUT) {
      float z = sAct[Offs<N, L - 1>::act + tid];
      if (N::kSigmoid) z = 1.f / (1.f + __expf(-z));
      out[(size_t)s * DOUT + tid] = z;
    }
    __syncthreads();
  }
}

using FFNNNet = Net<true, 10, 50, 30, 10, 1>;
using MLP64Net = Net<false, 10, 64, 64, 2>;
using TestingRemoteNet = Net<false, 2, 50, 10, 1>;
// autoencoder of the anomaly detector (models/mlp.py AE_SPEC): trained to reconstruct its input, MSE head.  Its instances
// are compiled in mlp_persistent_ae.cu, not here (see there).
using AENet = Net<false, 10, 32, 4, 32, 10>;
// attack-category classifier (models/mlp.py FFNN_CAT_SPEC): the FFNN's body with a 5-way linear head and softmax
// cross-entropy.  Its instances are compiled in mlp_persistent_cat.cu, for the reason mlp_persistent_ae.cu gives.
using CatNet = Net<false, 10, 50, 30, 10, 5>;

template <class N>
int smem_bytes(int batch_size) {
  using Tot = Totals<N>;
  int f = Tot::smem_params * (batch_size > 1 ? 2 : 1) + 3 * Tot::acts + 2 * CHUNK * Tot::ROW_MAX + 8;
  return f * (int)sizeof(float);
}

template <class N>
cudaError_t launch_t(const ClientDesc* descs, int n_clients, SgdHyper hp, cudaStream_t stream) {
  const int bytes = smem_bytes<N>(hp.batch_size);
  static int configured[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (bytes > configured[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(mlp_local_sgd_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return e;
    configured[dev & 63] = bytes;
  }
  COLEARN_LAUNCH(mlp_local_sgd_kernel<N>, n_clients, NT, bytes, stream, descs, hp);
  return cudaGetLastError();
}

template <class N>
cudaError_t forward_t(const float* theta, const float* x, float* out, int n, cudaStream_t stream) {
  using Tot = Totals<N>;
  const int bytes = (Tot::smem_params + N::DIN + Tot::acts + 8) * (int)sizeof(float);
  static bool configured[64] = {false};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!configured[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(mlp_forward_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return e;
    configured[dev & 63] = true;
  }
  int blocks = n < 132 * 2 ? n : 132 * 2;   // H100 SXM: 132 SMs
  if (blocks < 1) blocks = 1;
  COLEARN_LAUNCH(mlp_forward_kernel<N>, blocks, NT, bytes, stream, theta, x, out, n);
  return cudaGetLastError();
}

}  // namespace

#ifndef COLEARN_MLP_TEMPLATES_ONLY
// the autoencoder's instances (mlp_persistent_ae.cu): variants 1, 3, 5 and 6, the batched forward
cudaError_t launch_mlp_local_sgd_ae(const ClientDesc* descs, int n_clients, SgdHyper hp, cudaStream_t stream);
int mlp_local_sgd_smem_bytes_ae(int batch_size);
int mlp_net_num_params_ae();
cudaError_t launch_mlp_forward_ae(const float* theta, const float* x, float* out, int n, cudaStream_t stream);
// the attack-category FFNN's instances (mlp_persistent_cat.cu): variants 1, 3, 5 and 6, the batched forward
cudaError_t launch_mlp_local_sgd_cat(const ClientDesc* descs, int n_clients, SgdHyper hp, cudaStream_t stream);
int mlp_local_sgd_smem_bytes_cat(int batch_size);
int mlp_net_num_params_cat();
cudaError_t launch_mlp_forward_cat(const float* theta, const float* x, float* out, int n, cudaStream_t stream);

cudaError_t launch_mlp_local_sgd(int net_kind, const ClientDesc* descs, int n_clients, SgdHyper hp,
                                 cudaStream_t stream) {
  if (net_kind == NET_AE) return launch_mlp_local_sgd_ae(descs, n_clients, hp, stream);
  if (net_kind == NET_FFNN_CAT) return launch_mlp_local_sgd_cat(descs, n_clients, hp, stream);
  // variant 5 (default, set by ops/fused_mlp.py): register-resident weights, 128-thread CTA, blocked reduction slices
  // (LDS.128) + pre-scaled dz; 6: the same with its FMAs written in pairs; 3: the same kernel with strided slices;
  // 1: first version with smem-resident weights.
  if (hp.variant == 6) {
    switch (net_kind) {
      case NET_FFNN: return v2_128p::launch2<FFNNNet>(descs, n_clients, hp, stream);
      case NET_MLP64: return v2_128p::launch2<MLP64Net>(descs, n_clients, hp, stream);
      case NET_TESTING_REMOTE: return v2_128p::launch2<TestingRemoteNet>(descs, n_clients, hp, stream);
      default: return cudaErrorInvalidValue;
    }
  }
  if (hp.variant == 5) {
    switch (net_kind) {
      case NET_FFNN: return v2_128b::launch2<FFNNNet>(descs, n_clients, hp, stream);
      case NET_MLP64: return v2_128b::launch2<MLP64Net>(descs, n_clients, hp, stream);
      case NET_TESTING_REMOTE: return v2_128b::launch2<TestingRemoteNet>(descs, n_clients, hp, stream);
      default: return cudaErrorInvalidValue;
    }
  }
  if (hp.variant == 3) {
    switch (net_kind) {
      case NET_FFNN: return v2_128::launch2<FFNNNet>(descs, n_clients, hp, stream);
      case NET_MLP64: return v2_128::launch2<MLP64Net>(descs, n_clients, hp, stream);
      case NET_TESTING_REMOTE: return v2_128::launch2<TestingRemoteNet>(descs, n_clients, hp, stream);
      default: return cudaErrorInvalidValue;
    }
  }
  if (hp.variant != 1) return cudaErrorInvalidValue;
  switch (net_kind) {
    case NET_FFNN: return launch_t<FFNNNet>(descs, n_clients, hp, stream);
    case NET_MLP64: return launch_t<MLP64Net>(descs, n_clients, hp, stream);
    case NET_TESTING_REMOTE: return launch_t<TestingRemoteNet>(descs, n_clients, hp, stream);
    default: return cudaErrorInvalidValue;
  }
}

int mlp_local_sgd_smem_bytes(int net_kind, int batch_size) {
  switch (net_kind) {
    case NET_FFNN: return smem_bytes<FFNNNet>(batch_size);
    case NET_MLP64: return smem_bytes<MLP64Net>(batch_size);
    case NET_TESTING_REMOTE: return smem_bytes<TestingRemoteNet>(batch_size);
    case NET_AE: return mlp_local_sgd_smem_bytes_ae(batch_size);
    case NET_FFNN_CAT: return mlp_local_sgd_smem_bytes_cat(batch_size);
    default: return -1;
  }
}

int mlp_net_num_params(int net_kind) {
  switch (net_kind) {
    case NET_FFNN: return Totals<FFNNNet>::flat_params;
    case NET_MLP64: return Totals<MLP64Net>::flat_params;
    case NET_TESTING_REMOTE: return Totals<TestingRemoteNet>::flat_params;
    case NET_AE: return mlp_net_num_params_ae();
    case NET_FFNN_CAT: return mlp_net_num_params_cat();
    default: return -1;
  }
}

cudaError_t launch_mlp_forward(int net_kind, const float* theta, const float* x, float* out, int n,
                               cudaStream_t stream) {
  switch (net_kind) {
    case NET_FFNN: return forward_t<FFNNNet>(theta, x, out, n, stream);
    case NET_MLP64: return forward_t<MLP64Net>(theta, x, out, n, stream);
    case NET_TESTING_REMOTE: return forward_t<TestingRemoteNet>(theta, x, out, n, stream);
    case NET_AE: return launch_mlp_forward_ae(theta, x, out, n, stream);
    case NET_FFNN_CAT: return launch_mlp_forward_cat(theta, x, out, n, stream);
    default: return cudaErrorInvalidValue;
  }
}

COLEARN_DEFINE_SPIN_LIMIT_SETTER(set_spin_limit_mlp)
#endif  // COLEARN_MLP_TEMPLATES_ONLY

}  // namespace colearn
