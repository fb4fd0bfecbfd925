// Byzantine-robust aggregation (Yin et al., "Byzantine-Robust Distributed Learning", ICML 2018): coordinate-wise median
// and trimmed mean, formed per element inside the kernels that otherwise form the FedAvg average a = sum_k w_k theta_k:
// star_round_kernel and twoshot_chunk (comm.cu), fedavg_robust_kernel (elementwise.cu).  This is the only definition of
// the arithmetic; the GPU build and the SIMT CPU build (host_shim.h) both compile it.
//
// For one element with the n contributing values v_k in slot order:
//   key_k  = bits(v_k) ^ ((bits(v_k) >> 31) & 0x7fffffff), compared as int32 (IEEE total order: -NaN < -Inf < ... < -0 <
//            +0 < ... < +Inf < +NaN), ties broken by slot index:
//   rank_k = #{j : key_j < key_k} + #{j < k : key_j == key_k}
//   b      = floor((n - 1) / 2) (median) or min(floor(trim * n), floor((n - 1) / 2)) (trimmed mean; trim * n in float32)
//   a      = (sum over k in slot order of (b <= rank_k < n - b ? v_k : 0)) / (n - 2 b)      (IEEE division, no FMA)
// The robust kinds are unweighted.  ops/reference.py robust_aggregate is the PyTorch transcription.
// Included by colearn_kernels.h after COLEARN_HD is defined.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

namespace colearn {

enum AggKind : int { AGG_MEAN = 0, AGG_MEDIAN = 1, AGG_TRIMMED_MEAN = 2 };

// Zero-initialised (memset) = mean = the weighted FedAvg average: every existing caller keeps its path.
struct AggArgs {
  int kind;     // AggKind
  float trim;   // trimmed mean: fraction trimmed at each end, in [0, 0.5)
};

inline bool agg_args_ok(const AggArgs& g) {
  if (g.kind == AGG_MEAN || g.kind == AGG_MEDIAN) return true;
  return g.kind == AGG_TRIMMED_MEAN && g.trim >= 0.f && g.trim < 0.5f;
}

// values dropped at each end of the sorted n (>= 1) values
COLEARN_HD int agg_trim_count(const AggArgs& g, int n) {
  const int half = (n - 1) / 2;
  if (g.kind == AGG_MEDIAN) return half;
  const int b = (int)floorf(g.trim * (float)n);
  return b < half ? b : half;
}

COLEARN_HD int32_t agg_key(float v) {
#if defined(__CUDA_ARCH__)
  const int32_t bits = __float_as_int(v);
#else
  int32_t bits;
  memcpy(&bits, &v, sizeof(bits));
#endif
  return bits ^ ((bits >> 31) & 0x7fffffff);
}

// Register path: v[k] for the slots k set in `valid` (n = popcount(valid) >= 1; the other entries are ignored but must be
// initialised).  KMAX x KMAX compile-time-unrolled compares: the tie-break by slot index is the choice of <= (j < k) or < (j > k).
template <int KMAX>
COLEARN_HD float agg_robust(const float (&v)[KMAX], uint32_t valid, int n, int b) {
  int32_t key[KMAX];
#pragma unroll
  for (int k = 0; k < KMAX; ++k) key[k] = agg_key(v[k]);
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    int r = 0;
#pragma unroll
    for (int j = 0; j < KMAX; ++j) {
      if (j == k) continue;
      const bool before = (j < k) ? key[j] <= key[k] : key[j] < key[k];
      r += (before && ((valid >> j) & 1u)) ? 1 : 0;
    }
    const bool keep = ((valid >> k) & 1u) && b <= r && r < n - b;
    acc += keep ? v[k] : 0.f;
  }
  return acc / (float)(n - 2 * b);
}

// General path, any n >= 1, value k is ld(k): the values are taken TILE at a time into registers, in slot order, and each tile's
// ranks are counted against all n values streamed past it (j < tile: <=, j > tile: <, inside the tile: the register path's
// compile-time rule), so every value is read ceil(n / TILE) times instead of n times.  Same ranks, same summation order,
// same bits as agg_robust.
template <int TILE, class Load>
COLEARN_HD float agg_robust_tiled(const Load& ld, int n, int b) {
  float acc = 0.f;
  for (int t0 = 0; t0 < n; t0 += TILE) {
    float v[TILE];
    int32_t key[TILE];
    int r[TILE];
#pragma unroll
    for (int i = 0; i < TILE; ++i) {
      v[i] = (t0 + i < n) ? ld(t0 + i) : 0.f;
      key[i] = agg_key(v[i]);
    }
#pragma unroll
    for (int i = 0; i < TILE; ++i) {
      r[i] = 0;
#pragma unroll
      for (int j = 0; j < TILE; ++j) {
        if (j == i) continue;
        const bool before = (j < i) ? key[j] <= key[i] : key[j] < key[i];
        r[i] += (before && t0 + j < n) ? 1 : 0;
      }
    }
    for (int j = 0; j < t0; ++j) {
      const int32_t kj = agg_key(ld(j));
#pragma unroll
      for (int i = 0; i < TILE; ++i) r[i] += kj <= key[i] ? 1 : 0;
    }
    for (int j = t0 + TILE; j < n; ++j) {
      const int32_t kj = agg_key(ld(j));
#pragma unroll
      for (int i = 0; i < TILE; ++i) r[i] += kj < key[i] ? 1 : 0;
    }
#pragma unroll
    for (int i = 0; i < TILE; ++i) {
      const bool keep = t0 + i < n && b <= r[i] && r[i] < n - b;
      acc += keep ? v[i] : 0.f;
    }
  }
  return acc / (float)(n - 2 * b);
}

}  // namespace colearn
