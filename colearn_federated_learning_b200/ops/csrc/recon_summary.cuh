// Reconstruction-error summary of an autoencoder's outputs on held-out rows: per segment (one segment per device) additive
// integer counts — a histogram of the per-row error split by label — and a float64 error sum, from which fl/anomaly.py picks
// the federated alarm threshold and derives the detection metrics.  This is the only definition of the arithmetic; the GPU
// build and the SIMT CPU build (host_shim.h) both compile it, and ops/reference.py recon_summary is its bit-exact PyTorch
// transcription.  The work units, the shared-memory counts and the chunk order of the sum are eval_summary.cuh's.
//
// Inputs: xhat [N, D] fp32 (the model's output), x [N, D] fp32 (its input), labels [N] fp32 or none, segment offsets [S + 1].
//
// Error of a row (float64): e = sum_c d_c^2 over c = 0 .. D - 1 in column order from +0, d_c = xhat_c - x_c formed in fp32.
// d_c^2 is exact in float64 (a 24-bit significand squared), so contracting the adds into FMAs does not change a bit.
// Valid row: every value of xhat and x finite and, with labels, the label 0 or 1 (without labels every valid row counts as
// label 0).  Any other row counts only in n and n_invalid.
// Bin (from the bits of f = (float)e, no libm): B = 32 S bins, S = 2^s sub-bins per octave, 32 octaves [2^-24, 2^8):
//   f < 2^-24 (0 included): bin 0;  f >= 2^8: bin B - 1;  otherwise (E + 24) S + (top s bits of f's mantissa), E = f's exponent.
// Lower edge of bin j: 0 for j = 0, otherwise 2^(j / S - 24) (1 + (j mod S) / S); bin(e) >= j iff f >= that edge.
//
// Per segment, int64 words (rs_row_len(B) of them):
//   [0] n, [1] n_invalid, [2 + y B + b] histogram of the valid rows of label y in bin b
// Error sum: the valid rows' e in eval_summary.cuh's chunk order (2048-row chunks, 8 rows per thread in order, a butterfly
// over the warp, the 8 warps in order, the chunks of a segment in order, each from +0).
// Per-row outputs (optional): err[i] = (float)e, flag[i] = 1 iff the row is invalid or bin(e) >= alarm_bin.
// Limits: B a power of two in [32, 4096], 1 <= D <= 1024, N < 2^32 rows per launch (uint32 shared-memory counters), alarm_bin
// in [0, B].
// Included by colearn_kernels.h after eval_summary.cuh.
#pragma once
#include <stdint.h>
#include <string.h>

namespace colearn {

constexpr int kRsMinBins = 32;
constexpr int kRsMaxBins = 4096;
constexpr int kRsMaxDim = 1024;

COLEARN_HD int64_t rs_row_len(int bins) { return 2 + 2 * (int64_t)bins; }
// log2 of the sub-bins per octave, s = log2(B / 32)
COLEARN_HD int rs_sub_log2(int bins) {
  int s = 0;
  while ((kRsMinBins << s) < bins) ++s;
  return s;
}
COLEARN_HD uint32_t rs_float_bits(float f) {
#ifdef __CUDA_ARCH__
  return __float_as_uint(f);
#else
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
#endif
}
COLEARN_HD int rs_bin(double e, int sub_log2) {
  const uint32_t u = rs_float_bits((float)e);
  if (u < 0x33800000u) return 0;                                  // (float)e < 2^-24
  if (u >= 0x43800000u) return (kRsMinBins << sub_log2) - 1;      // (float)e >= 2^8
  return (int)(((u >> 23) - 103u) << sub_log2) + (int)((u & 0x7fffffu) >> (23 - sub_log2));
}

inline bool recon_summary_args_ok(int dim, int bins) {
  return dim >= 1 && dim <= kRsMaxDim && bins >= kRsMinBins && bins <= kRsMaxBins && (bins & (bins - 1)) == 0;
}

// Output block of one launch, int64 words: counts [S][rs_row_len] | err_sum [S] (float64) | ticket | partial [U] (float64, the
// chunk sums).  The launcher zeroes everything before partial.
COLEARN_HD int64_t rs_out_words(int segments, int bins, int64_t units) {
  return (int64_t)segments * rs_row_len(bins) + segments + 1 + units;
}

struct ReconSummaryArgs {
  const float* xhat;        // [N, D]
  const float* x;           // [N, D]
  const float* labels;      // [N] or nullptr
  const int64_t* table;     // es_build_table's words, device memory
  int segments;
  int64_t units;
  int dim;                  // D
  int bins;                 // B
  int alarm_bin;            // flag[i] = invalid || bin >= alarm_bin (read only with flag)
  float* err;               // [N] or nullptr
  uint8_t* flag;            // [N] or nullptr
  int64_t* out;             // rs_out_words(S, B, U) words, 8-byte aligned
};

}  // namespace colearn
