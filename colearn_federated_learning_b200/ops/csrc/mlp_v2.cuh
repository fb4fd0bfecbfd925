// Included three times by mlp_persistent.cu (V2_NS / V2_NT = CTA size, V2_BLOCKED, V2_PACKED), hence no include guard.  See the
// v2 header comment there.
namespace V2_NS {

constexpr int NT2 = V2_NT;
// V2_BLOCKED (variant 5): lane t of a neuron's lane group owns a CONTIGUOUS slice of the reduction index instead of every
// T-th element, so the 32-float slices of the 64-wide layers are fetched with 8 LDS.128 instead of 32 scalar LDS, and the
// producers of dz also publish scale * dz, so the column-copy update needs no FMUL per element.
#ifdef V2_BLOCKED
constexpr bool BLK = true;
#else
constexpr bool BLK = false;
#endif

// V2_PACKED (variant 6): the FMAs of the dot products and of the rank-1 updates are written as pairs on adjacent registers
// — same products, same order of additions per accumulator, so the results are bit-identical to the scalar form.  Hopper
// has no packed fp32 FMA: each pair compiles to two FFMA, and the variant computes what variant 5 computes.
#ifdef V2_PACKED
constexpr bool PK = true;
#else
constexpr bool PK = false;
#endif
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
// w[i] = fma(g, a[i], w[i]) for i < N (rank-1 update of a register slice)
template <int N>
__device__ __forceinline__ void axpy_regs(float (&w)[N], float g, const float (&a)[N]) {
  if constexpr (PK) {
    const float2 g2 = make_float2(g, g);
#pragma unroll
    for (int i = 0; i + 1 < N; i += 2) {
      const float2 r = fma2(g2, make_float2(a[i], a[i + 1]), make_float2(w[i], w[i + 1]));
      w[i] = r.x; w[i + 1] = r.y;
    }
    if constexpr (N & 1) w[N - 1] = fmaf(g, a[N - 1], w[N - 1]);
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i) w[i] = fmaf(g, a[i], w[i]);
  }
}
// accs[j] += w[4 q + j] * v[j], j < 4 (one 128-bit group of a blocked dot product; accumulator j keeps its own chain)
__device__ __forceinline__ void dot4(float (&accs)[4], const float* w, const float (&v)[4]) {
  if constexpr (PK) {
    const float2 r0 = fma2(make_float2(w[0], w[1]), make_float2(v[0], v[1]), make_float2(accs[0], accs[1]));
    const float2 r1 = fma2(make_float2(w[2], w[3]), make_float2(v[2], v[3]), make_float2(accs[2], accs[3]));
    accs[0] = r0.x; accs[1] = r0.y; accs[2] = r1.x; accs[3] = r1.y;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) accs[j] = fmaf(w[j], v[j], accs[j]);
  }
}

__host__ __device__ constexpr int gsize(int n_out, int k_in) {
  int t = pow2_floor(NT2 / n_out);
  if (t > 8) t = 8;   // <= 3 shuffle levels on the critical path
  while (t > 1 && t > k_in) t /= 2;
  return t;
}
__host__ __device__ constexpr int align4(int x) { return (x + 3) / 4 * 4; }

// Widest head that every warp replicates and fuses with its loss (HeadCfg::kFused, RL::REP).  The batch-1 instances hold such
// a head whole in every lane (HeadCfg::ht): DOUT x K weights, K inputs and DOUT biases, plus DOUT logits, exponentials and dz_L
// around the softmax, next to the row and column slices of the body.  On the FFNN body (10-50-30-10-C) ptxas fits every
// instance into its 255 registers without a spill up to C = 7; at C = 8 the batch-1 instances of variants 3, 5 and 6 spill.
// Hence 7: it covers the 5 attack categories with room, and the autoencoder's 10-wide head stays on the block-wide path.
constexpr int kFusedHeadMax = 7;

// Lanes per neuron of the set "outputs of layer LI" (LI <= L-2).  The SAME group size is used when that set is
// written (forward / row update of layer LI: T) and when its gradient is produced (dgrad of layer LI+1: TB),
// so thread (n, t) of layer LI's row copy is also the thread that holds dz for neuron n after the dgrad
// butterfly — the layer-0 update can take dz from a register instead of shared memory + a barrier.
template <class N, int LI>
__host__ __device__ constexpr int pair_group() {
  const int no = N::template dim<LI + 1>();
  int g = pow2_floor(NT2 / no);
  if (g > 8) g = 8;
  while (g > 1 && (g > N::template dim<LI>() || g > N::template dim<LI + 2>())) g /= 2;
  // In front of a fused softmax head (3 .. kFusedHeadMax classes) the group is capped so that a layer of <= 32 outputs fits
  // into one warp (RL::REP), as the loop above already does for heads of 1 or 2 outputs.  10-50-30-10-5: 2 lanes per neuron
  // of the 30 -> 10 layer, and 2 per input of the head's dgrad (one lane each needs 30 more registers for the row slices, and
  // the accumulating instances spill).
  if (LI == N::L - 2 && N::DOUT >= 3 && N::DOUT <= kFusedHeadMax && no <= 32 && g * no > 32) g = pow2_floor(32 / no);
  return g;
}
template <class N, int LI, bool HEAD = (LI == N::L - 1)>
struct GroupT { static constexpr int v = pair_group<N, LI>(); };
template <class N, int LI>
struct GroupT<N, LI, true> { static constexpr int v = gsize(N::template dim<LI + 1>(), N::template dim<LI>()); };
template <class N, int LI, bool FIRST = (LI == 0)>
struct GroupTB { static constexpr int v = pair_group<N, LI - 1>(); };
template <class N, int LI>
struct GroupTB<N, LI, true> { static constexpr int v = 1; };

template <class N, int LI>
struct RL {
  static constexpr int K = N::template dim<LI>();
  static constexpr int NO = N::template dim<LI + 1>();
  static constexpr int T = GroupT<N, LI>::v;
  static constexpr int KC = (K + T - 1) / T;
  // long row slices (the 64-thread CTA: one thread per neuron) re-read their inputs from shared memory in the update
  // instead of keeping them in registers from the forward pass (the activations are double-buffered, still valid)
  static constexpr bool KEEP = KC <= 32 || NT2 >= 128;   // (the measured 128 / 256-thread kernels keep everything)
  static constexpr int TB = GroupTB<N, LI>::v;
  static constexpr int NC = (NO + TB - 1) / TB;
  // Row copy replicated per warp: when the layer in front of the fused head fits into one warp (FFNN: 30 -> 10, ten threads), EVERY
  // warp computes all NO outputs itself — lane u owns the row slice thread u owned — and publishes them in its own slot of shared
  // memory, so the hop to the (per-warp) head needs __syncwarp instead of a block barrier: one of the step's barrier-separated
  // hops less, and no warp waits at a barrier for the one that used to do this layer alone.  The replicas stay identical: every
  // warp applies the same rank-1 update to its copy (same dz from shared memory, same inputs).
  static constexpr bool REP = (N::DOUT <= kFusedHeadMax) && (N::L >= 3) && (LI == N::L - 2) && (NO * T <= 32);
  static constexpr int RSTRIDE = (NO + 3) / 4 * 4;        // floats between the warps' output slots
  static __host__ __device__ constexpr int row_thread(int tid) { return REP ? (tid & 31) : tid; }
  // element i of lane t's row slice (reduction index k) / column slice (output index n)
  static constexpr bool KB = BLK && (K % T == 0);
  static constexpr bool NB = BLK && (NO % TB == 0);
  static __host__ __device__ constexpr int kidx(int i, int t) { return KB ? t * KC + i : i * T + t; }
  static __host__ __device__ constexpr int nidx(int i, int t) { return NB ? t * NC + i : i * TB + t; }
  // 128-bit shared-memory loads of a slice: activations / dz vectors start 16-byte aligned (AOff), samples do not
  static constexpr bool KV = KB && (KC % 4 == 0) && LI > 0;
  static constexpr bool NV = NB && (NC % 4 == 0);
  static constexpr int FW = Offs<N, LI>::flat;            // arena offset of W
  static constexpr int FB = Offs<N, LI>::flat + NO * K;   // arena offset of bias
};
// activation offsets padded to 16 bytes (a_{LI+1} lives at AOff<LI>)
template <class N, int LI> struct AOff {
  static constexpr int v = AOff<N, LI - 1>::v + (RL<N, LI - 1>::REP ? NT2 / 32 : 1) * align4(N::template dim<LI>());   // (one slot per warp)
};
template <class N> struct AOff<N, 0> { static constexpr int v = 0; };
template <class N> struct ATot { static constexpr int v = AOff<N, N::L>::v; };
// The head's column copy (dgrad of the head) follows the replication of the layer in front of it: every warp's lanes 0 .. K-1 own
// one input neuron each, write dz_{L-1} into the warp's own slot, and the dgrad of that layer reads it back after __syncwarp.
template <class N, int LI> struct ColRep { static constexpr bool v = (LI == N::L - 1) && RL<N, LI - 1>::REP; };
template <class N> struct ColRep<N, 0> { static constexpr bool v = false; };

template <class N> struct HeadCfg {
  static constexpr int LI = N::L - 1;
  static constexpr int K = N::template dim<LI>();
  static constexpr int DO = N::DOUT;
  // HT lanes share one dot product of the head (lane l owns inputs k = l % HT + HT * j); the 32 / HT groups of a warp compute the
  // same thing, and log2(HT) butterfly stages finish it; every stage (SHFL + FADD) sits on the step's dependent chain.
  // The 10-wide heads of the FFNN / 2-50-10-1 net are held whole in every lane (HT = 1: ten register FMAs, no shuffle); a
  // 64-wide head split 8 lanes x 8 inputs (3 stages instead of 5) spends on 16 extra loads and FMAs per lane what the two
  // stages save, so wide heads keep one lane per input.  The accumulating instances (batch > 1) have no registers to spare
  // and keep one lane per input, too.
  template <bool ACC> static constexpr int ht() { return (!ACC && K <= 16) ? 1 : 32; }
  template <bool ACC> static constexpr int kh() { return (K + ht<ACC>() - 1) / ht<ACC>(); }
  static constexpr int FW = Offs<N, LI>::flat;
  static constexpr int FB = Offs<N, LI>::flat + DO * K;
  static constexpr bool kFused = (N::DOUT <= kFusedHeadMax) && (N::L >= 2);
};

template <class N, int LI, bool ACC>
struct LayerRegs {
  float wr[RL<N, LI>::KC];
  float wt[RL<N, LI>::NC];
  float av[RL<N, LI>::KEEP ? RL<N, LI>::KC : 1];   // inputs of this thread's row slice, kept from forward to update
  float gr[ACC ? RL<N, LI>::KC : 1];
  float gt[ACC ? RL<N, LI>::NC : 1];
  float br, gb;
};
template <class N, int LI, bool ACC>
struct AllRegs : AllRegs<N, LI + 1, ACC> { LayerRegs<N, LI, ACC> r; };
template <class N, bool ACC>
struct AllRegs<N, N::L, ACC> {};
template <int LI, class N, bool ACC>
__device__ __forceinline__ LayerRegs<N, LI, ACC>& regs_of(AllRegs<N, 0, ACC>& all) {
  return static_cast<AllRegs<N, LI, ACC>&>(all).r;
}

template <class N, int LI, bool ACC>
__device__ __forceinline__ void load_regs(AllRegs<N, 0, ACC>& all, const float* __restrict__ theta, int tid) {
  using R = RL<N, LI>;
  auto& r = regs_of<LI>(all);
  if constexpr (!(HeadCfg<N>::kFused && LI == N::L - 1)) {   // the replicated head keeps its own row copy
    const int u = R::row_thread(tid);
    const int n = (u < R::NO * R::T) ? u / R::T : R::NO - 1, t = u % R::T;
#pragma unroll
    for (int i = 0; i < R::KC; ++i) {
      const int k = R::kidx(i, t);
      r.wr[i] = (k < R::K) ? __ldcg(theta + R::FW + n * R::K + k) : 0.f;
      if (ACC) r.gr[i] = 0.f;
    }
    r.br = __ldcg(theta + R::FB + n);
    r.gb = 0.f;
  }
  {
    const int uc = ColRep<N, LI>::v ? (tid & 31) : tid;
    const int k = (uc < R::K * R::TB) ? uc / R::TB : R::K - 1, t = uc % R::TB;
#pragma unroll
    for (int i = 0; i < R::NC; ++i) {
      const int n = R::nidx(i, t);
      r.wt[i] = (n < R::NO) ? __ldcg(theta + R::FW + n * R::K + k) : 0.f;
      if (ACC) r.gt[i] = 0.f;
    }
  }
  if constexpr (LI + 1 < N::L) load_regs<N, LI + 1, ACC>(all, theta, tid);
}

template <class N, int LI, bool ACC>
__device__ __forceinline__ void store_regs(AllRegs<N, 0, ACC>& all, const float* __restrict__ theta_in,
                                           float* __restrict__ theta_out, float w, int delta_mode, int tid) {
  using R = RL<N, LI>;
  auto& r = regs_of<LI>(all);
  if (!(HeadCfg<N>::kFused && LI == N::L - 1) && tid < R::NO * R::T) {
    const int n = tid / R::T, t = tid % R::T;
#pragma unroll
    for (int i = 0; i < R::KC; ++i) {
      const int k = R::kidx(i, t);
      if (k < R::K) {
        float v = r.wr[i];
        if (delta_mode) v -= __ldcg(theta_in + R::FW + n * R::K + k);
        theta_out[R::FW + n * R::K + k] = w * v;
      }
    }
    if (t == 0) {
      float v = r.br;
      if (delta_mode) v -= __ldcg(theta_in + R::FB + n);
      theta_out[R::FB + n] = w * v;
    }
  }
  if constexpr (LI + 1 < N::L) store_regs<N, LI + 1, ACC>(all, theta_in, theta_out, w, delta_mode, tid);
}

template <class N, int LI, bool ACC>
__device__ __forceinline__ void fwd(AllRegs<N, 0, ACC>& all, const float* __restrict__ a_in, float* __restrict__ a_out, int tid) {
  using R = RL<N, LI>;
  constexpr bool RELU = (LI != N::L - 1);
  auto& r = regs_of<LI>(all);
  const int u = R::row_thread(tid);
  const bool valid = u < R::NO * R::T;
  const int n = valid ? u / R::T : R::NO - 1, t = u % R::T;
  if constexpr (R::REP) a_out += (tid >> 5) * R::RSTRIDE;   // this warp's slot
  float accs[4] = {0.f, 0.f, 0.f, 0.f};
  if constexpr (BLK) accs[0] = (t == 0) ? r.br : 0.f;   // bias first: one dependent FADD less behind the shuffle
  if constexpr (R::KV) {
    // blocked slice: 128-bit loads of this lane's KC contiguous inputs
    const float4* p = reinterpret_cast<const float4*>(a_in + t * R::KC);
#ifdef COLEARN_HOST_SHIM
    if ((reinterpret_cast<uintptr_t>(p) & 15) != 0) abort();   // LDS.128 traps on a misaligned address
#endif
#pragma unroll
    for (int i4 = 0; i4 < R::KC / 4; ++i4) {
      const float4 v = p[i4];
      const float a4[4] = {v.x, v.y, v.z, v.w};
      if constexpr (R::KEEP) {
#pragma unroll
        for (int j = 0; j < 4; ++j) r.av[4 * i4 + j] = a4[j];
      }
      dot4(accs, &r.wr[4 * i4], a4);
    }
  } else {
#pragma unroll
    for (int i = 0; i < R::KC; ++i) {
      const int k = R::kidx(i, t);
      if constexpr (R::KEEP) {
        r.av[i] = (R::T * R::KC == R::K || k < R::K) ? a_in[k] : 0.f;
        accs[i & 3] = fmaf(r.wr[i], r.av[i], accs[i & 3]);
      } else {
        const float a = (R::T * R::KC == R::K || k < R::K) ? a_in[k] : 0.f;
        accs[i & 3] = fmaf(r.wr[i], a, accs[i & 3]);
      }
    }
  }
  float acc = (accs[0] + accs[1]) + (accs[2] + accs[3]);
#pragma unroll
  for (int o = R::T / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (valid && t == 0) {
    const float z = BLK ? acc : acc + r.br;
    a_out[n] = RELU ? relu_nan(z) : z;
  }
}

// blocked variant, batch 1: whoever produced dz_{LI+1} also published scale * dz_{LI+1} one ATot further, so the updates
// take the scaled value from shared memory (the same fp32 product scale * dz[n], computed once) instead of multiplying per
// element
template <class N, int LI, bool ACC>
struct ScaledIn { static constexpr bool v = BLK && !ACC && (HeadCfg<N>::kFused || LI < N::L - 1); };

// rank-1 update of the register copies of layer LI: the column copy (COL, LI >= 1; this lane's input neuron has activation
// ak, dzv = the dz_{LI+1} slice the dgrad read) and the row copy (ROW)
template <class N, int LI, bool ACC, bool COL = true, bool ROW = true>
__device__ __forceinline__ void update_copies(AllRegs<N, 0, ACC>& all, const float* __restrict__ dz_out, const float* __restrict__ a_in,
                                              const float (&dzv)[RL<N, LI>::NC], float ak, float scale, int tid) {
  using R = RL<N, LI>;
  auto& r = regs_of<LI>(all);
  constexpr bool SIN = ScaledIn<N, LI, ACC>::v;
  const float* sdz_out = dz_out + ATot<N>::v;
  if constexpr (LI > 0 && COL) {
    const int t = tid % R::TB;
    // column-copy update (same products, same order as the row copy below)
    if constexpr (SIN) {
      if constexpr (R::NV) {
        const float4* p = reinterpret_cast<const float4*>(sdz_out + t * R::NC);
#ifdef COLEARN_HOST_SHIM
        if ((reinterpret_cast<uintptr_t>(p) & 15) != 0) abort();   // LDS.128 traps on a misaligned address
#endif
#pragma unroll
        for (int i4 = 0; i4 < R::NC / 4; ++i4) {
          const float4 v = p[i4];
          if constexpr (PK) {
            const float2 ak2 = make_float2(ak, ak);
            const float2 r0 = fma2(make_float2(v.x, v.y), ak2, make_float2(r.wt[4 * i4], r.wt[4 * i4 + 1]));
            const float2 r1 = fma2(make_float2(v.z, v.w), ak2, make_float2(r.wt[4 * i4 + 2], r.wt[4 * i4 + 3]));
            r.wt[4 * i4] = r0.x; r.wt[4 * i4 + 1] = r0.y; r.wt[4 * i4 + 2] = r1.x; r.wt[4 * i4 + 3] = r1.y;
          } else {
            r.wt[4 * i4] = fmaf(v.x, ak, r.wt[4 * i4]);
            r.wt[4 * i4 + 1] = fmaf(v.y, ak, r.wt[4 * i4 + 1]);
            r.wt[4 * i4 + 2] = fmaf(v.z, ak, r.wt[4 * i4 + 2]);
            r.wt[4 * i4 + 3] = fmaf(v.w, ak, r.wt[4 * i4 + 3]);
          }
        }
      } else {
#pragma unroll
        for (int i = 0; i < R::NC; ++i) {
          const int n = R::nidx(i, t);
          const float sd = (R::TB * R::NC == R::NO || n < R::NO) ? sdz_out[n] : 0.f;
          r.wt[i] = fmaf(sd, ak, r.wt[i]);
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < R::NC; ++i) {
        if (ACC) r.gt[i] = fmaf(dzv[i], ak, r.gt[i]);
        else r.wt[i] = fmaf(scale * dzv[i], ak, r.wt[i]);
      }
    }
  }
  if constexpr (ROW) {
    const int u = R::row_thread(tid);
    const int n = (u < R::NO * R::T) ? u / R::T : R::NO - 1;
    const float d = SIN ? 0.f : dz_out[n];
    const float g = ACC ? d : (SIN ? sdz_out[n] : scale * d);
    if constexpr (R::KEEP) {
      if constexpr (ACC) axpy_regs(r.gr, g, r.av);
      else axpy_regs(r.wr, g, r.av);
    } else {
      const int t = u % R::T;
#pragma unroll
      for (int i = 0; i < R::KC; ++i) {
        const int k = R::kidx(i, t);
        const float a = (R::T * R::KC == R::K || k < R::K) ? a_in[k] : 0.f;
        if (ACC) r.gr[i] = fmaf(g, a, r.gr[i]);
        else r.wr[i] = fmaf(g, a, r.wr[i]);
      }
    }
    if (ACC) r.gb += g; else r.br += g;
  }
}

// backward of layer LI: dgrad (LI >= 1) from the thread-private column slices, then (UPDATE) the rank-1 update of
// both register copies.  No barrier between the two: the weights are private to the thread.  ak_out: the activation of this
// lane's input neuron, which the column-copy update multiplies with.
template <class N, int LI, bool ACC, bool WRITE_SMEM = true, bool UPDATE = true>
__device__ __forceinline__ float bwd(AllRegs<N, 0, ACC>& all, const float* __restrict__ dz_out, const float* __restrict__ a_in,
                                     float* __restrict__ dz_in, float scale, int tid, float* ak_out = nullptr) {
  using R = RL<N, LI>;
  auto& r = regs_of<LI>(all);
  float dz_mine = 0.f;   // dz of input neuron k = tid / TB, valid on every lane of the group (butterfly sum)
  float dzv[R::NC];
  float ak = 0.f;
  if constexpr (LI > 0) {
    const bool valid = tid < R::K * R::TB;
    const int k = valid ? tid / R::TB : R::K - 1, t = tid % R::TB;
    float accs[4] = {0.f, 0.f, 0.f, 0.f};
    if constexpr (R::NV) {
      const float4* p = reinterpret_cast<const float4*>(dz_out + t * R::NC);
#ifdef COLEARN_HOST_SHIM
      if ((reinterpret_cast<uintptr_t>(p) & 15) != 0) abort();   // LDS.128 traps on a misaligned address
#endif
#pragma unroll
      for (int i4 = 0; i4 < R::NC / 4; ++i4) {
        const float4 v = p[i4];
        dzv[4 * i4] = v.x; dzv[4 * i4 + 1] = v.y; dzv[4 * i4 + 2] = v.z; dzv[4 * i4 + 3] = v.w;
        const float d4[4] = {v.x, v.y, v.z, v.w};
        dot4(accs, &r.wt[4 * i4], d4);
      }
    } else {
#pragma unroll
      for (int i = 0; i < R::NC; ++i) {
        const int n = R::nidx(i, t);
        dzv[i] = (R::TB * R::NC == R::NO || n < R::NO) ? dz_out[n] : 0.f;
        accs[i & 3] = fmaf(r.wt[i], dzv[i], accs[i & 3]);
      }
    }
    float acc = (accs[0] + accs[1]) + (accs[2] + accs[3]);
#pragma unroll
    for (int o = R::TB / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    ak = a_in[k];
    dz_mine = relu_grad(ak, acc);
    if (WRITE_SMEM && valid && t == 0) {
      dz_in[k] = dz_mine;
      if constexpr (BLK && !ACC) dz_in[k + ATot<N>::v] = scale * dz_mine;
    }
  }
  if constexpr (UPDATE) update_copies<N, LI, ACC>(all, dz_out, a_in, dzv, ak, scale, tid);
  if (ak_out) *ak_out = ak;
  return dz_mine;
}

// layer-0 row update with dz taken from a register (see pair_group): no shared memory, no barrier
template <class N, bool ACC>
__device__ __forceinline__ void bwd0_from_reg(AllRegs<N, 0, ACC>& all, float dz_reg, float scale) {
  using R = RL<N, 0>;
  static_assert(R::KEEP, "the layer-0 row slice keeps its inputs in registers");
  auto& r = regs_of<0>(all);
  const float g = ACC ? dz_reg : scale * dz_reg;
  if constexpr (ACC) axpy_regs(r.gr, g, r.av);
  else axpy_regs(r.wr, g, r.av);
  if (ACC) r.gb += g; else r.br += g;
}

// Batch 1: the rank-1 updates of layer 1 that bwd<1> left out (ROW: the row copy, COL: the column copy), issued during the NEXT
// step (docs/KERNELS.md §2).  They read dz_2 (and scale * dz_2) from sDz / this warp's slot, which that step does not
// overwrite before its second block barrier (or, per warp, its first __syncwarp), the row inputs from r.av and the column
// input a_1[k] from ak (a register: the activation buffer of the previous parity is rewritten by the step after next, which
// the 2-50-10-1 net reaches without another block barrier).
template <class N, bool COL, bool ROW>
__device__ __forceinline__ void bwd1_deferred(AllRegs<N, 0, false>& all, float ak, const float* dzs, float scale, int tid) {
  using R = RL<N, 1>;
  static_assert(R::KEEP, "the row update takes its inputs from registers");
  const float* dz_out = dzs + AOff<N, 1>::v + (R::REP ? (tid >> 5) * R::RSTRIDE : 0);
  const int t = tid % R::TB;
  float dzv[R::NC];
  if constexpr (COL && !ScaledIn<N, 1, false>::v) {
#pragma unroll
    for (int i = 0; i < R::NC; ++i) {
      const int n = R::nidx(i, t);
      dzv[i] = (R::TB * R::NC == R::NO || n < R::NO) ? dz_out[n] : 0.f;
    }
  }
  update_copies<N, 1, false, COL, ROW>(all, dz_out, nullptr, dzv, ak, scale, tid);
}

template <class N, int LI, bool ACC>
__device__ __forceinline__ void apply_grads(AllRegs<N, 0, ACC>& all, float neg_lr) {
  using R = RL<N, LI>;
  auto& r = regs_of<LI>(all);
#pragma unroll
  for (int i = 0; i < R::KC; ++i) { r.wr[i] = fmaf(neg_lr, r.gr[i], r.wr[i]); r.gr[i] = 0.f; }
#pragma unroll
  for (int i = 0; i < R::NC; ++i) { r.wt[i] = fmaf(neg_lr, r.gt[i], r.wt[i]); r.gt[i] = 0.f; }
  r.br = fmaf(neg_lr, r.gb, r.br);
  r.gb = 0.f;
  if constexpr (LI + 1 < N::L) apply_grads<N, LI + 1, ACC>(all, neg_lr);
}


// ---- replicated head (DOUT <= kFusedHeadMax) ---------------------------------------------------------------------
// Every warp keeps its own copy of the head layer (HeadCfg::ht lanes per dot product).  After the
// barrier that publishes a_{L-1}, each warp computes the logits itself (register FMAs + a short butterfly), so
// every thread knows dz_L in registers: the "head -> loss -> barrier -> dgrad" hop of the step disappears
// (4 instead of 5 barrier-separated dependency hops per SGD step).
template <class N, bool ACC>
struct HeadRegs {
  static constexpr int HT = HeadCfg<N>::template ht<ACC>(), KH = HeadCfg<N>::template kh<ACC>();
  float wh[HeadCfg<N>::DO][KH];
  float ah[KH];
  float bh[HeadCfg<N>::DO];
  float gh[ACC ? HeadCfg<N>::DO : 1][ACC ? KH : 1];
  float gbh[ACC ? HeadCfg<N>::DO : 1];
};

template <class N, bool ACC>
__device__ __forceinline__ void head_load(HeadRegs<N, ACC>& H, const float* __restrict__ theta, int lane) {
  using C = HeadCfg<N>;
  constexpr int HT = HeadRegs<N, ACC>::HT, KH = HeadRegs<N, ACC>::KH;
#pragma unroll
  for (int c = 0; c < C::DO; ++c) {
#pragma unroll
    for (int j = 0; j < KH; ++j) {
      const int k = (lane & (HT - 1)) + HT * j;
      H.wh[c][j] = (k < C::K) ? __ldcg(theta + C::FW + c * C::K + k) : 0.f;
      if (ACC) H.gh[c][j] = 0.f;
    }
    H.bh[c] = __ldcg(theta + C::FB + c);
    if (ACC) H.gbh[c] = 0.f;
  }
}
template <class N, bool ACC>
__device__ __forceinline__ void head_store(const HeadRegs<N, ACC>& H, const float* __restrict__ theta_in,
                                           float* __restrict__ theta_out, float w, int delta_mode, int tid) {
  using C = HeadCfg<N>;
  constexpr int HT = HeadRegs<N, ACC>::HT, KH = HeadRegs<N, ACC>::KH;
  if (tid < HT) {                      // (the first group of warp 0: one owner per input)
#pragma unroll
    for (int c = 0; c < C::DO; ++c) {
#pragma unroll
      for (int j = 0; j < KH; ++j) {
        const int k = tid + HT * j;
        if (k < C::K) {
          float v = H.wh[c][j];
          if (delta_mode) v -= __ldcg(theta_in + C::FW + c * C::K + k);
          theta_out[C::FW + c * C::K + k] = w * v;
        }
      }
      if (tid == 0) {
        float v = H.bh[c];
        if (delta_mode) v -= __ldcg(theta_in + C::FB + c);
        theta_out[C::FB + c] = w * v;
      }
    }
  }
}

// exp(x) for x <= 0 and 1 / x for a normal x > 0 as single MUFU instructions (ex2.approx.ftz, rcp.approx.ftz: 2 ulp / 1 ulp, the
// latter over every normal argument).  The heads call them on the step's dependent chain with x in [1, 2] (the sigmoid's 1 + e)
// and in [1, C] (the softmax sum of a C-class head): __expf adds a range fix-up around MUFU.EX2, __frcp_rn a Newton step and a
// slow-path branch around MUFU.RCP — neither can trigger for these arguments.
#ifdef COLEARN_HOST_SHIM
inline float exp_nonpos(float x) { return expf(x); }
inline float rcp_approx(float x) { return 1.0f / x; }
#else
__device__ __forceinline__ float exp_nonpos(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x * 1.4426950408889634f));
  return r;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
#endif

// logits (all-reduced inside every warp) -> dz_L in registers of every thread; returns the loss (valid on tid 0)
template <class N, bool ACC>
__device__ __forceinline__ float head_forward_loss(HeadRegs<N, ACC>& H, const float* __restrict__ a_in,
                                                   const float* __restrict__ yrow, int loss, float inv_b,
                                                   float (&dzh)[HeadCfg<N>::DO], int lane, int tid) {
  using C = HeadCfg<N>;
  float z[C::DO];
#pragma unroll
  for (int c = 0; c < C::DO; ++c) z[c] = 0.f;
  constexpr int HT = HeadRegs<N, ACC>::HT, KH = HeadRegs<N, ACC>::KH;
  if constexpr (HT == 1) {
    // the whole input vector in every lane: 16-byte broadcast loads (a_{L-1} starts 16-byte aligned: AOff), two partial sums
    static_assert(KH == C::K, "one lane holds every input");
#pragma unroll
    for (int q = 0; q < C::K / 4; ++q) {
      const float4 v = reinterpret_cast<const float4*>(a_in)[q];
      H.ah[4 * q] = v.x; H.ah[4 * q + 1] = v.y; H.ah[4 * q + 2] = v.z; H.ah[4 * q + 3] = v.w;
    }
#pragma unroll
    for (int k = (C::K / 4) * 4; k < C::K; ++k) H.ah[k] = a_in[k];
    float z2[C::DO];
#pragma unroll
    for (int c = 0; c < C::DO; ++c) z2[c] = 0.f;
#pragma unroll
    for (int j = 0; j < KH; ++j) {
#pragma unroll
      for (int c = 0; c < C::DO; ++c) {
        if (j & 1) z2[c] = fmaf(H.wh[c][j], H.ah[j], z2[c]);
        else z[c] = fmaf(H.wh[c][j], H.ah[j], z[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < C::DO; ++c) z[c] += z2[c];
  } else {
#pragma unroll
    for (int j = 0; j < KH; ++j) {
      const int k = (lane & (HT - 1)) + HT * j;
      H.ah[j] = (KH * HT == C::K || k < C::K) ? a_in[k] : 0.f;
#pragma unroll
      for (int c = 0; c < C::DO; ++c) z[c] = fmaf(H.wh[c][j], H.ah[j], z[c]);
    }
#pragma unroll
    for (int o = HT / 2; o > 0; o >>= 1) {
#pragma unroll
      for (int c = 0; c < C::DO; ++c) z[c] += __shfl_xor_sync(0xffffffffu, z[c], o);
    }
  }
#pragma unroll
  for (int c = 0; c < C::DO; ++c) z[c] += H.bh[c];
  float value = 0.f;
  if (loss == LOSS_XENT) {
    const int label = (int)yrow[0];
    if constexpr (C::DO >= 3) {
      // softmax cross-entropy, in every thread's registers: m = max z, e_c = exp(z_c - m), s = sum e_c in [1, DO],
      // dz_c = (e_c / s - [c == y]) / B, loss log(s) + m - z_y.  z_y by compare-and-select over the compile-time class
      // index (a dynamically indexed register array would go to local memory).
      float m = z[0];
#pragma unroll
      for (int c = 1; c < C::DO; ++c) m = fmaxf(m, z[c]);
      float e[C::DO], s = 0.f, zy = 0.f;
#pragma unroll
      for (int c = 0; c < C::DO; ++c) {
        e[c] = exp_nonpos(z[c] - m);
        s += e[c];
        zy = (label == c) ? z[c] : zy;
      }
      const float r = rcp_approx(s);   // s in [1, DO]
#pragma unroll
      for (int c = 0; c < C::DO; ++c) dzh[c] = (e[c] * r - (label == c ? 1.f : 0.f)) * inv_b;
      value = (__logf(s) + m) - zy;   // (every thread: see below)
    } else {
      const float d = (C::DO == 2) ? z[C::DO - 1] - z[0] : 0.f;
      const float e = exp_nonpos(-fabsf(d));
      const float r1 = rcp_approx(1.f + e);
      const float p1 = d >= 0.f ? r1 : e * r1;
      dzh[0] = ((1.f - p1) - (label == 0 ? 1.f : 0.f)) * inv_b;
      if (C::DO == 2) dzh[C::DO - 1] = (p1 - (label == 1 ? 1.f : 0.f)) * inv_b;
      {  // (every thread, no branch: the value only feeds the loss statistics, so it schedules off the dependent chain, while an
         //  `if (tid == 0)` made warp 0 run MUFU.LG2 + a reconvergence point in front of the barrier the other warps wait at)
        const float margin = (label == 0) ? d : -d;
        value = fmaxf(margin, 0.f) + __logf(1.f + e);
      }
    }
  } else {
#pragma unroll
    for (int c = 0; c < C::DO; ++c) {
      const float y = yrow[c], zz = z[c];
      if (N::kSigmoid) {
        const float e = exp_nonpos(-fabsf(zz));
        const float r1 = rcp_approx(1.f + e);
        const float out = zz >= 0.f ? r1 : e * r1;
        if (loss == LOSS_BCE) {
          dzh[c] = (out - y) * inv_b * (1.f / C::DO);
          value += (fmaxf(zz, 0.f) + __logf(1.f + e) - y * zz) * (1.f / C::DO);
        } else {
          const float df = out - y;
          dzh[c] = 2.f * df * out * (1.f - out) * ((loss == LOSS_MSE) ? inv_b : 1.f);
          value += df * df;
        }
      } else {
        const float df = zz - y;
        dzh[c] = 2.f * df * ((loss == LOSS_MSE) ? inv_b : 1.f);
        value += df * df;
      }
    }
  }
  return value;
}

// rank-1 update of this warp's replicated head copy (inputs H.ah of the step that produced dzh)
template <class N, bool ACC>
__device__ __forceinline__ void head_update(HeadRegs<N, ACC>& H, const float (&dzh)[HeadCfg<N>::DO], float scale) {
  using C = HeadCfg<N>;
#pragma unroll
  for (int c = 0; c < C::DO; ++c) {
    const float g = ACC ? dzh[c] : scale * dzh[c];
#pragma unroll
    for (int j = 0; j < HeadRegs<N, ACC>::KH; ++j) {
      if (ACC) H.gh[c][j] = fmaf(g, H.ah[j], H.gh[c][j]);
      else H.wh[c][j] = fmaf(g, H.ah[j], H.wh[c][j]);
    }
    if (ACC) H.gbh[c] += g; else H.bh[c] += g;
  }
}

// backward of the replicated head: dgrad for a_{L-1} from the column copies (wt) + dz_L registers, update of
// the column copies and (UPDATE_HEAD) of every warp's replicated head copy.
template <class N, bool ACC, bool UPDATE_HEAD = true>
__device__ __forceinline__ void head_backward(AllRegs<N, 0, ACC>& all, HeadRegs<N, ACC>& H,
                                              const float (&dzh)[HeadCfg<N>::DO], const float* __restrict__ a_in,
                                              float* __restrict__ dz_in, float scale, int tid) {
  using C = HeadCfg<N>;
  using R = RL<N, C::LI>;
  auto& r = regs_of<C::LI>(all);
  constexpr bool CR = ColRep<N, C::LI>::v;
  const int uc = CR ? (tid & 31) : tid;
  const bool valid = uc < R::K * R::TB;
  const int k = valid ? uc / R::TB : R::K - 1, t = uc % R::TB;
  if constexpr (CR) dz_in += (tid >> 5) * RL<N, C::LI - (C::LI > 0)>::RSTRIDE;   // this warp's slot
  float dzv[R::NC];
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < R::NC; ++i) {
    const int n = R::nidx(i, t);
    if constexpr (C::DO >= 3) {   // dz_n by compare-and-select over the class index (n >= DO: a padding slot, 0)
      float v = 0.f;
#pragma unroll
      for (int c = 0; c < C::DO; ++c) v = (n == c) ? dzh[c] : v;
      dzv[i] = v;
    } else {
      dzv[i] = (n == 0) ? dzh[0] : ((C::DO == 2 && n == 1) ? dzh[C::DO - 1] : 0.f);
    }
    acc = fmaf(r.wt[i], dzv[i], acc);
  }
#pragma unroll
  for (int o = R::TB / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  const float ak = a_in[k];
  if (valid && t == 0) {
    const float dzk = relu_grad(ak, acc);
    dz_in[k] = dzk;
    if constexpr (BLK && !ACC) dz_in[k + ATot<N>::v] = scale * dzk;   // see bwd(): SIN
  }
#pragma unroll
  for (int i = 0; i < R::NC; ++i) {
    if (ACC) r.gt[i] = fmaf(dzv[i], ak, r.gt[i]);
    else r.wt[i] = fmaf(scale * dzv[i], ak, r.wt[i]);
  }
  if constexpr (UPDATE_HEAD) head_update<N, ACC>(H, dzh, scale);
}
template <class N, bool ACC>
__device__ __forceinline__ void head_apply_grads(HeadRegs<N, ACC>& H, float neg_lr) {
  using C = HeadCfg<N>;
#pragma unroll
  for (int c = 0; c < C::DO; ++c) {
#pragma unroll
    for (int j = 0; j < HeadRegs<N, ACC>::KH; ++j) { H.wh[c][j] = fmaf(neg_lr, H.gh[c][j], H.wh[c][j]); H.gh[c][j] = 0.f; }
    H.bh[c] = fmaf(neg_lr, H.gbh[c], H.bh[c]);
    H.gbh[c] = 0.f;
  }
}

template <class N, int LI, bool ACC>
struct Fwd2 {
  // runs layers LI .. LAST-1 (each followed by a barrier); LAST = L-1 when the head is fused with the loss
  static constexpr int LAST = HeadCfg<N>::kFused ? N::L - 1 : N::L;
  static __device__ __forceinline__ void run(AllRegs<N, 0, ACC>& all, const float* a0, float* acts, int tid) {
    if constexpr (LI < LAST) {
      const float* a_in = (LI == 0) ? a0 : acts + AOff<N, LI - (LI > 0)>::v;
      fwd<N, LI, ACC>(all, a_in, acts + AOff<N, LI>::v, tid);
      if constexpr (RL<N, LI>::REP) __syncwarp();     // the consumer is this warp's own head
      else __syncthreads();
      Fwd2<N, LI + 1, ACC>::run(all, a0, acts, tid);
    }
  }
};

// DEFER1 (batch 1): layer 1's rank-1 updates are left to bwd1_deferred
template <class N, int LI, bool ACC, bool DEFER1 = false>
struct Bwd2 {
  static __device__ __forceinline__ void run(AllRegs<N, 0, ACC>& all, const float* a0, const float* acts, float* dzs,
                                             float scale, int tid, float* ak1 = nullptr) {
    const float* a_in = (LI == 0) ? a0 : acts + AOff<N, LI - (LI > 0)>::v;
    float* dz_in = dzs + AOff<N, LI - (LI > 0)>::v;   // dz_{LI} (unused for LI == 0)
    const float* dz_out = dzs + AOff<N, LI>::v + (RL<N, LI>::REP ? (tid >> 5) * RL<N, LI>::RSTRIDE : 0);   // dz_{LI+1} (REP: own slot)
    if constexpr (LI == 1) {
      // dz_1 stays in registers: the thread pair that reduces dz_1[n] is the pair that owns row n of layer 0
      static_assert(RL<N, 1>::TB == RL<N, 0>::T && RL<N, 1>::K == RL<N, 0>::NO, "layer-0/1 lane mappings must coincide");
      const float dz1 = bwd<N, 1, ACC, false, !DEFER1>(all, dz_out, a_in, dz_in, scale, tid, ak1);
      bwd0_from_reg<N, ACC>(all, dz1, scale);
    } else {
      bwd<N, LI, ACC>(all, dz_out, a_in, dz_in, scale, tid);
      if constexpr (LI > 0) {
        __syncthreads();   // dz_{LI} visible to the next layer's threads
        Bwd2<N, LI - 1, ACC, DEFER1>::run(all, a0, acts, dzs, scale, tid, ak1);
      }
    }
  }
};

// single-thread loss for tiny heads (DOUT <= 2): no shuffles on the critical path
template <class N>
__device__ __forceinline__ float loss_small(float* aL, float* dzL, const float* yrow, int loss, float inv_b) {
  constexpr int DO = N::DOUT;
  if (loss == LOSS_XENT) {
    const int label = (int)yrow[0];
    float m = aL[0];
#pragma unroll
    for (int j = 1; j < DO; ++j) m = fmaxf(m, aL[j]);
    float e[DO], s = 0.f;
#pragma unroll
    for (int j = 0; j < DO; ++j) { e[j] = __expf(aL[j] - m); s += e[j]; }
    const float inv_s = 1.f / s;
    float zl = 0.f;
#pragma unroll
    for (int j = 0; j < DO; ++j) {
      dzL[j] = (e[j] * inv_s - (j == label ? 1.f : 0.f)) * inv_b;
      if (j == label) zl = aL[j];
    }
    return (__logf(s) + m) - zl;
  }
  float value = 0.f;
#pragma unroll
  for (int j = 0; j < DO; ++j) {
    const float z = aL[j], y = yrow[j];
    float out = z, dact = 1.f;
    if (N::kSigmoid) { out = 1.f / (1.f + __expf(-z)); dact = out * (1.f - out); }
    if (loss == LOSS_BCE) {
      const float lp = fmaxf(__logf(out), -100.f), l1p = fmaxf(log1pf(-out), -100.f);
      value -= (y * lp + (1.f - y) * l1p) * (1.f / DO);
      dzL[j] = (out - y) * inv_b * (1.f / DO);
    } else {
      const float d = out - y;
      value += d * d;
      dzL[j] = 2.f * d * dact * ((loss == LOSS_MSE) ? inv_b : 1.f);
    }
  }
  return value;
}

// Staged model (flat layout, shared memory; already scaled) -> theta_out as 16-byte vectors.  Out of line on purpose: it runs
// once per fit, and inlined its loops changed the register allocation and the schedule of the training loop above it.
__device__ COLEARN_NOINLINE void write_out_staged(const float* sOut, float* theta_out, int P, int tid) {
  int e0 = 0;
  if ((reinterpret_cast<uintptr_t>(theta_out) & 15) == 0) {
    for (int q = tid; q < P / 4; q += NT2) reinterpret_cast<float4*>(theta_out)[q] = reinterpret_cast<const float4*>(sOut)[q];
    e0 = (P / 4) * 4;
  }
  for (int e = e0 + tid; e < P; e += NT2) theta_out[e] = sOut[e];
}

// floats of dynamic shared memory in front of the write-out staging area (activations, dz, two data chunks, loss cells, the
// index ring), rounded up so that the staging area can be read as float4
template <class N>
__host__ __device__ constexpr int stage_offset2() {
  return (((BLK ? 4 : 3) * ATot<N>::v + 2 * CHUNK * Totals<N>::ROW_MAX + 8 + 2 * CHUNK) + 3) / 4 * 4;
}

template <class N, bool ACC>
__global__ void __launch_bounds__(NT2, 1)
mlp_local_sgd_kernel_v2(const ClientDesc* __restrict__ descs, SgdHyper hp) {
  using Tot = Totals<N>;
  constexpr int DIN = N::DIN, ROWM = Tot::ROW_MAX;
  constexpr int EPT2 = (CHUNK * ROWM + NT2 - 1) / NT2;
  constexpr int ACTS = ATot<N>::v;
  COLEARN_DYN_SMEM(float, smem);
  const ClientDesc d = descs[blockIdx.x];
  const int tid = threadIdx.x;
  const int B = hp.batch_size < 1 ? 1 : hp.batch_size;

  float* sAct = smem;                       // 2 x ACTS (double buffered by step parity)
  float* sDz = sAct + 2 * ACTS;             // ACTS (blocked variant: + ACTS of scale * dz right behind)
  float* sData = sDz + (BLK ? 2 : 1) * ACTS;   // 2 x CHUNK x ROWM
  float* sMisc = sData + 2 * CHUNK * ROWM;  // [0] last loss, [1] loss sum
  // Two forms of the gather's index lookup, chosen per net (docs/KERNELS.md §2): RING = one thread per sample resolves the
  // index two chunks ahead into a shared-memory ring (the 4-layer nets, with the keyed order computed right there); otherwise
  // every gathering thread reads the order table itself (the 64-wide MLP)
  constexpr bool RING = (N::L >= 4);
  int* sIdx = reinterpret_cast<int*>(sMisc + 8);   // RING: 2 x CHUNK sample indices

  const int n = d.n, ydim = d.y_dim, row = DIN + ydim;
  // An empty shard (trailing virtual clients of a short one, see shard_bounds) gets Q = 0 (spe counts it as one step per
  // epoch of 0 samples): no steps and no loads from x, y or perm; the write-out stores out_scale * theta_in (0 in delta
  // mode), the losses are {0, 0}, the flags work as usual.
  const int spe = ((n > 0 ? n : 1) + B - 1) / B;
  long long total_steps = (long long)hp.epochs * spe;
  if (hp.max_steps > 0 && hp.max_steps < total_steps) total_steps = hp.max_steps;
  long long Q;
  {
    const long long full_epochs = total_steps / spe;
    long long rem_samples = (total_steps - full_epochs * spe) * B;
    if (rem_samples > n) rem_samples = n;
    Q = full_epochs * (long long)n + rem_samples;
  }
  const int n_chunks = (int)((Q + CHUNK - 1) / CHUNK);

  // Sample order.  d.perm: a caller-made table.  d.perm_seed: the kernel makes the table ITSELF, right here — all threads
  // fill d.perm_scratch with the keyed Feistel bijection of every epoch this fit will touch (the shuffle of the reference's
  // loaders: no separate launch, no host round trip, and it runs while the broadcast this client waits for is still in
  // flight).  The gather below then reads either table with plain (coherent) loads.
  const int* perm_tab = d.perm;
  int perm_rows = d.perm_rows;
  const FeistelDomain fdom = feistel_domain((uint32_t)(n > 0 ? n : 1));
  if (!RING && d.perm == nullptr && d.perm_seed != 0 && d.perm_scratch != nullptr && n > 0) {
    const int rows = (int)((Q + n - 1) / n);
    const long long total = (long long)rows * n;
    for (long long e = tid; e < total; e += NT2) {
      const int r = (int)(e / n);
      d.perm_scratch[e] = (int)feistel_index((uint32_t)(e - (long long)r * n), (uint32_t)n, fdom, d.perm_seed, d.perm_row0 + r);
    }
    __syncthreads();
    perm_tab = d.perm_scratch;
    perm_rows = rows > 0 ? rows : 1;
  }
  // only now wait for this round's broadcast and pull the model into registers
  if (d.wait_flag != nullptr) {
    if (tid == 0) spin_wait_ge(d.wait_flag, d.wait_value, 32, "mlp_local_sgd: broadcast flag of this round");
    __syncthreads();
  }
  AllRegs<N, 0, ACC> W;
  load_regs<N, 0, ACC>(W, d.theta_in, tid);
  HeadRegs<N, ACC> H;
  if constexpr (HeadCfg<N>::kFused) head_load<N, ACC>(H, d.theta_in, tid & 31);
  if (tid < 2) sMisc[tid] = 0.f;
  float last_loss = 0.f, loss_sum = 0.f;   // blocked variant and batch 1: thread 0 keeps the loss statistics in registers (it is their only reader)
  auto sample_index = [&](long long q) -> int {
    const int ep = (int)(q / n);
    const int pos = (int)(q - (long long)ep * n);
    if (perm_tab) return __ldcg(perm_tab + (size_t)(ep % perm_rows) * n + pos);
    if (RING && d.perm_seed) return (int)feistel_index((uint32_t)pos, (uint32_t)n, fdom, d.perm_seed, d.perm_row0 + ep);
    return pos;
  };
  auto compute_indices = [&](int chunk) {      // RING only: threads 0 .. CHUNK-1, one sample each
    if (tid < CHUNK) {
      const long long q = (long long)chunk * CHUNK + tid;
      sIdx[(chunk & 1) * CHUNK + tid] = q < Q ? sample_index(q) : 0;
    }
  };
  float pre[EPT2];
  auto issue_loads = [&](int chunk) {
    const int* order = sIdx + (chunk & 1) * CHUNK;
#pragma unroll
    for (int j = 0; j < EPT2; ++j) {
      const int e = tid + j * NT2;
      pre[j] = 0.f;
      if (e < CHUNK * row) {
        const int i = e / row, c = e - i * row;
        const long long q = (long long)chunk * CHUNK + i;
        if (q < Q) {
          const int idx = RING ? order[i] : sample_index(q);
          pre[j] = (c < DIN) ? __ldg(d.x + (size_t)idx * DIN + c) : __ldg(d.y + (size_t)idx * ydim + (c - DIN));
        }
      }
    }
  };
  auto store_loads = [&](int buf) {
    float* dst = sData + buf * (CHUNK * ROWM);
#pragma unroll
    for (int j = 0; j < EPT2; ++j) {
      const int e = tid + j * NT2;
      if (e < CHUNK * row) dst[e] = pre[j];
    }
  };
  if constexpr (RING) {
    if (n_chunks > 0) compute_indices(0);
    if (n_chunks > 1) compute_indices(1);
    __syncthreads();
  }
  if (n_chunks > 0) { issue_loads(0); store_loads(0); }
  __syncthreads();

  long long step = 0;
  int pos_in_epoch = 0, in_batch = 0;
  int cur_batch = (n < B) ? n : B;
  float batch_loss = 0.f;
  int parity = 0;
  const float neg_lr = -hp.lr;
  // Batch 1 (ACC == false): every sample is an SGD step, so the step body carries none of the batch bookkeeping, and the rank-1
  // updates that nothing on the dependent chain waits for — both copies of layer 1 and the head — move out of the tail of their
  // step, where they stood in-order between dz_1 and the next step's first loads (docs/KERNELS.md §2):
  //   * the row copy of layer 1 and the head go to the top of the next step, in one basic block with the layer-0 forward, and
  //     fill the latency of its sample loads (layer 1's forward reads the row copy right after the first barrier);
  //   * the column copy of layer 1 goes behind that barrier, where its loads and FMAs fill the latency of the layer-1 forward
  //     and the head (its first reader is the dgrad of layer 1).
  // Same operands, same FMA per weight: the model is bit-identical.  The first step of a chunk has nothing pending; the last
  // one's updates are issued after the chunk's steps.
  constexpr bool DEFER = !ACC && HeadCfg<N>::kFused && N::L >= 3;
  float dzh_last[HeadCfg<N>::DO];   // batch 1: dz_L of the last step (DEFER: its head update is pending)
#pragma unroll
  for (int j = 0; j < HeadCfg<N>::DO; ++j) dzh_last[j] = 0.f;
  float ak1_last = 0.f;              // DEFER: a_1[k] of the last step, input of the pending column-copy update
  auto deferred_before_fwd0 = [&]() {
    if constexpr (DEFER) {
      bwd1_deferred<N, false, true>(W, 0.f, sDz, neg_lr, tid);
      head_update<N, ACC>(H, dzh_last, neg_lr);
    }
  };
  auto deferred_after_fwd0 = [&]() {
    if constexpr (DEFER) bwd1_deferred<N, true, false>(W, ak1_last, sDz, neg_lr, tid);
  };

  for (int c = 0; c < n_chunks; ++c) {
    if (c + 1 < n_chunks) issue_loads(c + 1);
    if constexpr (RING) {
      if (c + 2 < n_chunks) compute_indices(c + 2);      // slot c & 1: chunk c's indices were consumed one iteration ago
    }
    const float* chunk = sData + (c & 1) * (CHUNK * ROWM);
    const long long q0 = (long long)c * CHUNK;
    const int cnt = (int)((Q - q0) < CHUNK ? (Q - q0) : CHUNK);
    if constexpr (!ACC) {
      auto train_step = [&](auto pending, int i) {
        if constexpr (decltype(pending)::value) deferred_before_fwd0();
        const float* a0 = chunk + i * row;
        float* acts = sAct + parity * ACTS;
        static_assert(!RL<N, 0>::REP, "layer 0 publishes its outputs through a block barrier");
        fwd<N, 0, ACC>(W, a0, acts + AOff<N, 0>::v, tid);
        __syncthreads();
        if constexpr (decltype(pending)::value) deferred_after_fwd0();
        Fwd2<N, 1, ACC>::run(W, a0, acts, tid);
        float v = 0.f;
        if constexpr (HeadCfg<N>::kFused) {
          constexpr int LH = N::L - 1;
          const float* a_head = acts + AOff<N, LH - 1>::v + (RL<N, LH - 1>::REP ? (tid >> 5) * RL<N, LH - 1>::RSTRIDE : 0);
          v = head_forward_loss<N, ACC>(H, a_head, a0 + DIN, hp.loss, 1.f, dzh_last, tid & 31, tid);
          head_backward<N, ACC, !DEFER>(W, H, dzh_last, a_head, sDz + AOff<N, LH - 1>::v, neg_lr, tid);
          if constexpr (RL<N, LH - 1>::REP) __syncwarp();
          else __syncthreads();
          Bwd2<N, LH - 1, ACC, DEFER>::run(W, a0, acts, sDz, neg_lr, tid, &ak1_last);
        } else {
          if (tid < 32) v = loss_and_dz<N>(acts + AOff<N, N::L - 1>::v, sDz + AOff<N, N::L - 1>::v, a0 + DIN, hp.loss, 1.f, tid);
          __syncthreads();
          Bwd2<N, N::L - 1, ACC>::run(W, a0, acts, sDz, neg_lr, tid);
        }
        parity ^= 1;
        const float step_loss = 0.f + v;   // the sum the batch path forms (a -0 loss reports as +0); thread 0's copy is reported
        last_loss = step_loss;
        loss_sum += step_loss;
      };
      if constexpr (DEFER) {
        train_step(std::false_type{}, 0);
        for (int i = 1; i < cnt; ++i) train_step(std::true_type{}, i);
        deferred_before_fwd0();
        deferred_after_fwd0();
      } else {
        for (int i = 0; i < cnt; ++i) train_step(std::false_type{}, i);
      }
    } else for (int i = 0; i < cnt; ++i) {
      const float* a0 = chunk + i * row;
      float* acts = sAct + parity * ACTS;
      const float inv_b = 1.f / (float)cur_batch;

      Fwd2<N, 0, ACC>::run(W, a0, acts, tid);
      if constexpr (HeadCfg<N>::kFused) {
        constexpr int LH = N::L - 1;
        // a_{L-1}, published by the last barrier (or by this warp itself: RL::REP)
        const float* a_head = acts + AOff<N, LH - 1>::v + (RL<N, LH - 1>::REP ? (tid >> 5) * RL<N, LH - 1>::RSTRIDE : 0);
        float dzh[HeadCfg<N>::DO];
        const float v = head_forward_loss<N, ACC>(H, a_head, a0 + DIN, hp.loss, inv_b, dzh, tid & 31, tid);
        batch_loss += (hp.loss == LOSS_SSE) ? v : v * inv_b;     // (all threads: thread 0's copy is the one that is reported)
        head_backward<N, ACC>(W, H, dzh, a_head, sDz + AOff<N, LH - 1>::v, neg_lr, tid);
        if constexpr (RL<N, LH - 1>::REP) __syncwarp();            // dz_{L-1}: this warp's slot, read back by this warp
        else __syncthreads();                                      // dz_{L-1} visible
        Bwd2<N, LH - 1, ACC>::run(W, a0, acts, sDz, neg_lr, tid);
      } else {
        if (tid < 32) {
          const float v = loss_and_dz<N>(acts + AOff<N, N::L - 1>::v, sDz + AOff<N, N::L - 1>::v, a0 + DIN, hp.loss, inv_b, tid);
          if (tid == 0) batch_loss += (hp.loss == LOSS_SSE) ? v : v * inv_b;
        }
        __syncthreads();
        Bwd2<N, N::L - 1, ACC>::run(W, a0, acts, sDz, neg_lr, tid);
      }
      parity ^= 1;

      ++in_batch;
      ++pos_in_epoch;
      if (in_batch == cur_batch) {
        if (ACC) { apply_grads<N, 0, ACC>(W, neg_lr); if constexpr (HeadCfg<N>::kFused) head_apply_grads<N, ACC>(H, neg_lr); }
        if (BLK) { last_loss = batch_loss; loss_sum += batch_loss; batch_loss = 0.f; }
        else if (tid == 0) { sMisc[0] = batch_loss; sMisc[1] += batch_loss; batch_loss = 0.f; }
        ++step;
        in_batch = 0;
        if (pos_in_epoch >= n) pos_in_epoch = 0;
        const int left = n - pos_in_epoch;
        cur_batch = left < B ? left : B;
      }
    }
    __syncthreads();
    if (c + 1 < n_chunks) store_loads((c + 1) & 1);
    __syncthreads();
  }
  if constexpr (!ACC) step = Q;
  __syncthreads();
  // Write-out.  The registers hold the model in the layers' lane mappings (lane t of a row owns a blocked or strided slice of
  // it): stored from there, every 4-byte store is its own 32-byte NVLink packet when theta_out is a coordinator's slot on
  // another GPU.  STAGED: the same stores (scale and delta included) target a staging area in shared memory — a generic
  // pointer, same ST.E instructions — and the model leaves as 16-byte vectors, 512 contiguous bytes per warp instruction.
  // ptxas schedules the training loop of the 64-wide MLP differently as soon as this epilogue changes, so the 3-layer nets
  // keep the direct stores.
  constexpr bool STAGED = (N::L >= 4);
  if constexpr (STAGED) {
    float* sOut = smem + stage_offset2<N>();
    store_regs<N, 0, ACC>(W, d.theta_in, sOut, d.out_scale, d.delta_mode, tid);
    if constexpr (HeadCfg<N>::kFused) head_store<N, ACC>(H, d.theta_in, sOut, d.out_scale, d.delta_mode, tid);
    __syncthreads();
    write_out_staged(sOut, d.theta_out, Tot::flat_params, tid);
  } else {
    store_regs<N, 0, ACC>(W, d.theta_in, d.theta_out, d.out_scale, d.delta_mode, tid);
    if constexpr (HeadCfg<N>::kFused) head_store<N, ACC>(H, d.theta_in, d.theta_out, d.out_scale, d.delta_mode, tid);
  }
  if (tid == 0 && d.loss_out != nullptr) {
    constexpr bool REG = BLK || !ACC;   // loss statistics kept in registers
    d.loss_out[0] = REG ? last_loss : sMisc[0];
    d.loss_out[1] = step > 0 ? (REG ? loss_sum : sMisc[1]) / (float)step : 0.f;
  }
  __syncthreads();
  if (tid == 0 && d.signal_flag != nullptr) {
    __threadfence_system();
    st_release_sys(d.signal_flag, d.signal_value);
  }
}

template <class N>
int smem_bytes2() {
  return (stage_offset2<N>() + (N::L >= 4 ? Totals<N>::flat_params + 4 : 0)) * (int)sizeof(float);
}
template <class N>
cudaError_t launch2(const ClientDesc* descs, int n_clients, SgdHyper hp, cudaStream_t stream) {
  const int bytes = smem_bytes2<N>();
  // (launched through a pointer: a template-id with a comma cannot travel through the launch macro)
  void (*kern)(const ClientDesc*, SgdHyper) = hp.batch_size > 1 ? mlp_local_sgd_kernel_v2<N, true> : mlp_local_sgd_kernel_v2<N, false>;
  COLEARN_LAUNCH(kern, n_clients, NT2, bytes, stream, descs, hp);
  return cudaGetLastError();
}

}  // namespace V2_NS
