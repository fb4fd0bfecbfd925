// Weighted distance-based robust aggregation: every row k of the K client rows x_k is reweighted by its L2 distance d_k from a
// centre and the aggregate is a weighted mean.  Two kinds:
//   geomed     the geometric median of RFA (Pillutla, Kakade, Harchaoui, "Robust Aggregation for Federated Learning", IEEE TSP
//              2022): L smoothed Weiszfeld steps from the start point c^0
//   norm_clip  the start point plus the alpha-weighted sum of the updates, each clipped to L2 norm tau (Sun et al., "Can You
//              Really Backdoor Federated Learning?", 2019)
// This is the only definition of the arithmetic; the GPU build and the SIMT CPU build (host_shim.h) both compile it, and
// ops/reference.py distance_aggregate is its PyTorch transcription.
//
// Rows and start point: fp32 rows are the client models and c^0 = theta; int8 / int4 rows are the decoded deltas, c^0 = 0 and
// theta is added to the aggregate at the end.  alpha_k: the FedAvg weights of the caller.
//
// Distance.  d_k(c) = sqrt(sum_j (x_k[j] - c[j])^2): the difference in float32, its square accumulated in float64 with explicit
// fma.  The sum runs over fixed chunks of kDaChunk = 2048 elements (one 256-thread CTA x 8 elements per lane: lane l of warp w
// holds elements 2048 q + 256 w + 8 l + i, i = 0..7).  Inside a chunk: a lane sums its 8 squares in order i = 0..7 from +0, the
// 32 lanes of a warp are added by a halving tree (lane l + lane l + o for o = 16, 8, 4, 2, 1), and the 8 warp sums are added in
// warp order.  Over the chunks: lane t of one CTA adds the chunk sums q = t, t + 256, ... in ascending order from +0, and the 256
// lane sums are added as inside a chunk.  The partition does not depend on the launch grid, so neither does any result.
//
// Weights.  A row whose d_k is not finite is excluded: its weight is exactly 0 and the sums select it out (a NaN / Inf never
// enters a sum).  With the rows left (all float64, sums in row order):
//   geomed     beta_k = alpha_k / max(eps, d_k), B = sum beta_k, w_k = (float)(beta_k / B)
//   norm_clip  A = sum alpha_k, w_k = (float)(alpha_k / A * min(1, tau / d_k))
// When no row is left, or B / A is not > 0, every w_k is 0 and the aggregate is the start point.
//
// Centre and aggregate (float32, fmaf in row order from +0, rows of weight 0 skipped):
//   geomed     c^l[j] = sum_k fmaf(w_k(c^{l-1}), x_k[j], acc), l = 1..L;     a = c^L
//   norm_clip  a[j] = c^0[j] + sum_k fmaf(w_k(c^0), x_k[j] - c^0[j], acc)
// a is then theta + a for deltas, and theta moves towards it by opt.lr or the server optimizer step (server_opt.cuh).
// Included by colearn_kernels.h after COLEARN_HD is defined.
#pragma once
#include <math.h>
#include <stdint.h>

namespace colearn {

enum DistAggKind : int { DAGG_GEOMED = 3, DAGG_NORM_CLIP = 4 };   // after the AggKind codes (robust_agg.cuh)

constexpr int kDaThreads = 256;
constexpr int kDaChunk = kDaThreads * 8;
constexpr int kDaMaxIters = 16;

struct DistAggArgs {
  int kind;     // DistAggKind
  int iters;    // geomed: L in 1..16
  float eps;    // geomed: nu, finite and > 0
  float clip;   // norm_clip: tau, finite and > 0
};

inline bool dist_agg_args_ok(const DistAggArgs& g) {
  if (g.kind == DAGG_GEOMED) return g.iters >= 1 && g.iters <= kDaMaxIters && g.eps > 0.f && g.eps < INFINITY;
  return g.kind == DAGG_NORM_CLIP && g.clip > 0.f && g.clip < INFINITY;
}

COLEARN_HD int64_t da_chunks(int64_t n) { return (n + kDaChunk - 1) / kDaChunk; }

// Scratch of one aggregation (caller-owned, no state between calls): the per-row chunk sums, the per-row distances,
// the raw and final weights of the current step and the ticket of the finalisation.  da_scratch_bytes(k, n) bytes, 16-byte aligned.
struct DistAggScratch {
  double* partial;     // [k][da_chunks(n)]
  double* dist;        // [k]: d_k
  double* raw;         // [k]: da_raw of row k
  float* w;            // [k]
  unsigned* ticket;    // [1], zeroed by the launcher, left at 0 by the last CTA
  int* live;           // [1], rows with a weight > 0
};
inline int64_t da_scratch_bytes(int k, int64_t n) {
  const int64_t kk = ((int64_t)k + 1) & ~(int64_t)1;
  return (int64_t)8 * kk * da_chunks(n) + 16 * kk + 4 * kk + 16;
}
inline DistAggScratch da_scratch_carve(void* base, int k, int64_t n) {
  const int64_t kk = ((int64_t)k + 1) & ~(int64_t)1;
  char* p = static_cast<char*>(base);
  DistAggScratch s;
  s.partial = reinterpret_cast<double*>(p);
  p += 8 * kk * da_chunks(n);
  s.dist = reinterpret_cast<double*>(p);
  p += 8 * kk;
  s.raw = reinterpret_cast<double*>(p);
  p += 8 * kk;
  s.w = reinterpret_cast<float*>(p);
  p += 4 * kk;
  s.ticket = reinterpret_cast<unsigned*>(p);
  s.live = reinterpret_cast<int*>(p + 4);
  return s;
}

// a lane's 8 squared differences in order, float32 difference, float64 fma
COLEARN_HD double da_lane_sq8(const float (&x)[8], const float (&c)[8]) {
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const double d = (double)(x[i] - c[i]);
    s = fma(d, d, s);
  }
  return s;
}

// The weights, per row from its distance d (NaN / Inf: excluded).  raw: beta_k (geomed) or alpha_k (norm_clip), 0 for an
// excluded row; the caller sums them in row order into tot, and when tot > 0 the weight is da_weight, otherwise 0.
COLEARN_HD bool da_kept(double d) { return d < INFINITY; }    // false for NaN
COLEARN_HD double da_raw(const DistAggArgs& g, float alpha, double d) {
  if (!da_kept(d)) return 0.0;
  return g.kind == DAGG_GEOMED ? (double)alpha / fmax((double)g.eps, d) : (double)alpha;
}
COLEARN_HD float da_weight(const DistAggArgs& g, double raw, double d, double tot) {
  if (!da_kept(d)) return 0.f;
  return g.kind == DAGG_GEOMED ? (float)(raw / tot) : (float)(raw / tot * fmin(1.0, (double)g.clip / d));
}

}  // namespace colearn
