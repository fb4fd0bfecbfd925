// Detection-metrics summary of a model's outputs on held-out rows: additive integer counts (confusion matrix, score
// histograms) and a float64 loss sum per segment (one segment per device), from which fl/fedeval.py derives accuracy,
// detection / false-alarm rates, precision, F1, ROC-AUC and average precision.  This is the only definition of the
// arithmetic; the GPU build and the SIMT CPU build (host_shim.h) both compile it, and ops/reference.py eval_summary is its
// PyTorch transcription.
//
// Inputs: scores [N, C] fp32 (the model outputs after its output activation: probabilities for C = 1, logits for C >= 2),
// labels [N] fp32, segment offsets [S + 1] (0 = o_0 <= o_1 <= ... <= o_S = N).  C' = 2 when C = 1, otherwise C.
//
// Valid row: every score finite, for C = 1 also in [0, 1], and the label an integer k with 0 <= k < C'.  Any other row counts
// only in n and n_invalid.
//
// Per segment, int64 words (es_row_len(C, B) of them):
//   [0] n, [1] n_invalid
//   [2 + C' t + p]                     confusion: true class t, predicted class p
//   [2 + C'^2 + (2 h + pos) B + b]     histogram h < C (H = C) of the score p_h, pos = 1 for the rows whose label is the
//                                      positive class (C = 1: y == 1; C >= 2: y == h), bin b < B
// Prediction: C = 1 positive iff p > threshold; C >= 2 argmax of the scores, lowest index among equals.
// Score of histogram h: C = 1 the output p itself; C >= 2 the softmax p_h = e_h / sum_c e_c, e_c = exp((double)z_c - m),
// m = max_c z_c, computed in float64 (the class sum in class order).
// Bin: b = min(B - 1, (int)(p B)), B a power of two in [2, 4096]: for a float p, p B is exact in fp32; for the float64
// softmax a bin edge is only crossed by a difference in the last bit of a float64 exp, so every build gives the same bins.
// Loss of a valid row (float64): C = 1 the BCE -log(p) (y = 1) or -log1p(-p) (y = 0) with each log floored at -100 as torch's
// binary_cross_entropy does (bce_log_floor); C >= 2 the cross-entropy log(sum_c e_c) - ((double)z_y - m).
// Loss order: a segment is cut into chunks of kEsChunk = 2048 rows.  Thread t of a 256-thread CTA sums the rows t, t + 256,
// ..., t + 1792 of a chunk in that order from +0, the 32 lanes of a warp are added by a butterfly (xor 16, 8, 4, 2, 1) and the
// 8 warp sums in warp order; the chunk sums of a segment are added in chunk order from +0.  The partition depends neither on
// the launch grid nor on the other segments of a launch.
// Limits: 1 <= C <= 32, C 2 B <= 32768 (the histograms of a CTA live in shared memory as uint32 counters), N < 2^32 rows per
// launch (a CTA's counters are flushed only when it changes segment, so with one CTA a segment's whole count sits in one uint32;
// the bindings refuse more rows).
// Included by colearn_kernels.h after COLEARN_HD is defined.
#pragma once
#include <math.h>
#include <stdint.h>

#include <vector>

namespace colearn {

constexpr int kEsThreads = 256;
constexpr int kEsChunk = 2048;
constexpr int kEsRowsPerThread = kEsChunk / kEsThreads;
constexpr int kEsMaxClasses = 32;
constexpr int kEsMinBins = 2;
constexpr int kEsMaxBins = 4096;
constexpr int kEsMaxHistWords = 32768;
constexpr int64_t kEsMaxRows = ((int64_t)1 << 32) - 1;

COLEARN_HD int es_classes(int c) { return c == 1 ? 2 : c; }
COLEARN_HD int64_t es_conf_off() { return 2; }
COLEARN_HD int64_t es_hist_off(int c) { return 2 + (int64_t)es_classes(c) * es_classes(c); }
COLEARN_HD int64_t es_row_len(int c, int bins) { return es_hist_off(c) + (int64_t)c * 2 * bins; }
COLEARN_HD int64_t es_chunks(int64_t rows) { return (rows + kEsChunk - 1) / kEsChunk; }

inline bool eval_summary_args_ok(int c, int bins, float threshold) {
  const bool pow2 = bins >= kEsMinBins && bins <= kEsMaxBins && (bins & (bins - 1)) == 0;
  return c >= 1 && c <= kEsMaxClasses && pow2 && (int64_t)c * 2 * bins <= kEsMaxHistWords && threshold >= 0.f && threshold <= 1.f;
}

// the label as a class index, or -1 when the row is not valid for it (NaN, negative, fractional, >= C')
COLEARN_HD int es_label(float y, int c) {
  return (y >= 0.f && y < (float)es_classes(c) && y == floorf(y)) ? (int)y : -1;
}
COLEARN_HD int es_bin(float p, int bins) {
  const int b = (int)(p * (float)bins);
  return b < bins - 1 ? b : bins - 1;
}
COLEARN_HD int es_bin(double p, int bins) {
  const int b = (int)(p * (double)bins);
  return b < bins - 1 ? b : bins - 1;
}
COLEARN_HD double es_log_floor(double x) { return x < -100.0 ? -100.0 : x; }
// BCE of a valid C = 1 row
COLEARN_HD double es_bce(float p, int label) {
  return label == 1 ? -es_log_floor(log((double)p)) : -es_log_floor(log1p(-(double)p));
}

// Work units of one launch: (segment, chunk) pairs in segment order.  table = offsets [S + 1] | unit_seg [U] | seg_unit0 [S + 1]
// (the first unit of each segment, U at the end), int64 words; returns U, or -1 for offsets that are not 0 = o_0 <= ... <= o_S.
inline int64_t es_build_table(const int64_t* offsets, int segments, std::vector<int64_t>& table) {
  if (segments < 1 || offsets[0] != 0) return -1;
  int64_t units = 0;
  for (int s = 0; s < segments; ++s) {
    if (offsets[s + 1] < offsets[s]) return -1;
    units += es_chunks(offsets[s + 1] - offsets[s]);
  }
  table.assign(offsets, offsets + segments + 1);
  for (int s = 0; s < segments; ++s)
    for (int64_t q = 0; q < es_chunks(offsets[s + 1] - offsets[s]); ++q) table.push_back(s);
  int64_t u = 0;
  for (int s = 0; s < segments; ++s) {
    table.push_back(u);
    u += es_chunks(offsets[s + 1] - offsets[s]);
  }
  table.push_back(u);
  return units;
}

// Output block of one launch, int64 words: counts [S][es_row_len] | loss [S] (float64) | ticket | partial [U] (float64, the
// chunk sums).  The launcher zeroes everything before partial.
COLEARN_HD int64_t es_out_words(int segments, int c, int bins, int64_t units) {
  return (int64_t)segments * es_row_len(c, bins) + segments + 1 + units;
}

struct EvalSummaryArgs {
  const float* scores;      // [N, C], any 4-byte alignment
  const float* labels;      // [N]
  const int64_t* table;     // es_build_table's words, device memory
  int segments;
  int64_t units;
  int classes;              // C
  int bins;                 // B
  float threshold;          // C = 1: positive iff p > threshold
  int64_t* out;             // es_out_words(S, C, B, U) words, 8-byte aligned
};

}  // namespace colearn
