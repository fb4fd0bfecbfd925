// Top-k sparsified uplink with error feedback (EF-SGD: Seide et al. 2014, Stich et al. 2018, Karimireddy et al. 2019): a
// client keeps the k largest-magnitude entries of every 256-element block of v = d + e (its delta d = theta_k - theta plus the
// residual e it did not send in earlier rounds), sends them as (uint8 offset, fp32 value) pairs and carries the rest over.
// topk_delta_kernel (encode) and fedavg_topk_kernel (decode fused into the FedAvg apply) in elementwise.cu use these
// functions, and so do the top-k downlink kernels (downlink.cuh); the GPU build and the SIMT CPU build (host_shim.h) both
// compile them, and ops/reference.py encode_topk_delta / decode_topk_delta is the numpy transcription.
//
// Per element j (fp32, in this order and with no other arithmetic):  d_j = m_j - theta_j,  v_j = d_j + e_j.
// Blocks are the codec's kUqBlock-element blocks: block b covers [256 b, min(256 b + 256, P)), length m_b; it keeps
// k_b = min(k, m_b) entries (1 <= k <= kUtMaxK).
//   key a_j = |v_j| bit pattern as uint32, every NaN mapped to 0x7f800001 (the GPU writes a canonical NaN, the CPU keeps
//             payloads: one key keeps both ranking alike); NaN and Inf sort above every finite value, so they are always kept
//   kept    = the k_b elements with the greatest key, the lower j winning ties
//   wire    = per block, k_b uint8 offsets j - 256 b in ascending order and their fp32 values v_j, blocks packed one after the
//             other: block b < nblk - 1 starts at entry b k, E(P, k) = k (nblk - 1) + min(k, m_last) entries in all
//   e_j    <- 0 for the kept elements, v_j for the others (sent + new residual == v bit for bit)
// Decode + aggregate: per element acc = +0, then for each slot c in slot order that sent j, acc = fmaf(w_c, value, acc);
// a = theta + acc and the server step towards a.
// Included by colearn_kernels.h after uplink_quant.cuh.
#pragma once
#include <stdint.h>

namespace colearn {

constexpr int kUtMaxK = 32;                 // at most one entry per lane of the warp that owns a block

// the selection key of v
COLEARN_HD uint32_t ut_key(float v) {
  const uint32_t a = uq_abs_bits(v);
  return a > 0x7f800000u ? 0x7f800001u : a;
}

// entries of a row of n elements at k per block
COLEARN_HD int64_t ut_entries(int64_t n, int k) {
  const int64_t nblk = uq_nblk(n);
  const int64_t last = n - (nblk - 1) * kUqBlock;
  return (int64_t)k * (nblk - 1) + (last < k ? last : k);
}

// entries kept in block blk
COLEARN_HD int ut_block_k(int64_t n, int64_t blk, int k) {
  const int64_t m = n - blk * kUqBlock;
  return m < k ? (int)m : k;
}

}  // namespace colearn
