// Secure aggregation of the device updates (Bonawitz et al., CCS 2017): pairwise-masked fixed-point deltas in the ring of uint32.
// secagg_mask_kernel (a device masks its update), fedavg_secagg_kernel / secagg_streams_kernel (the coordinator removes the
// masks that did not cancel, decodes the sum and applies the mean) in elementwise.cu use these functions; the GPU build and the
// SIMT CPU build (host_shim.h) both compile them, and ops/reference.py chacha20_blocks / secagg_mask / secagg_unmask_sum /
// secagg_decode is the numpy transcription.  fl/secagg.py holds the protocol.
//
// Streams: stream s with 32-byte key k (8 little-endian uint32 words) is the ChaCha20 keystream of RFC 8439 with nonce 0:
// element e is word e mod 16 of block counter = e / 16.  A row of P elements takes ceil(P / 16) blocks: P < 2^36.
// Encode (a device, delta d = model - theta, clip C, fraction bits f):
//   NaN -> 0 (counted non-finite); +-Inf -> +-C (counted non-finite); |d| > C -> +-C (counted clipped)
//   q = __float2int_rn(clamp(d, -C, C) * 2^f)     (the product is exact: 2^f is a power of two; round half to even)
//   y = q + sum_s sign_s PRG(k_s)  (mod 2^32)      sign_s = +1 or -1
// Decode (the coordinator, the survivors' sum z of the q, |U2| = n):
//   mean = __fdiv_rn((float)(int32)z * 2^-f, (float)n)          (int -> float rounds to nearest even, then exact scaling)
// and theta moves towards a = theta + mean (apply8<OPT> of elementwise.cu).  f is chosen so that |U1| ceil(C 2^f) <= 2^31 - 1:
// no honest sum wraps.  Whatever a device sends, |mean| <= 2^31 2^-f / n.
// Included by colearn_kernels.h after COLEARN_HD is defined.
#pragma once
#include <math.h>
#include <stdint.h>

namespace colearn {

constexpr int kSaWords = 16;                             // uint32 words of one ChaCha20 block: the elements one thread owns
constexpr int64_t kSaMaxElems = (int64_t)1 << 36;        // the block counter is one uint32 word

COLEARN_HD uint32_t sa_rotl(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }

COLEARN_HD void sa_quarter(uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d) {
  a += b; d ^= a; d = sa_rotl(d, 16);
  c += d; b ^= c; b = sa_rotl(b, 12);
  a += b; d ^= a; d = sa_rotl(d, 8);
  c += d; b ^= c; b = sa_rotl(b, 7);
}

// RFC 8439 §2.3: the 16 output words of the block `counter` of key k (8 words) and nonce (n0, n1, n2)
COLEARN_HD void sa_chacha20_block(const uint32_t (&k)[8], uint32_t counter, uint32_t n0, uint32_t n1, uint32_t n2,
                                  uint32_t (&out)[kSaWords]) {
  uint32_t x[kSaWords] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, k[0], k[1], k[2], k[3],
                          k[4], k[5], k[6], k[7], counter, n0, n1, n2};
#pragma unroll 1
  for (int r = 0; r < 10; ++r) {
    sa_quarter(x[0], x[4], x[8], x[12]);
    sa_quarter(x[1], x[5], x[9], x[13]);
    sa_quarter(x[2], x[6], x[10], x[14]);
    sa_quarter(x[3], x[7], x[11], x[15]);
    sa_quarter(x[0], x[5], x[10], x[15]);
    sa_quarter(x[1], x[6], x[11], x[12]);
    sa_quarter(x[2], x[7], x[8], x[13]);
    sa_quarter(x[3], x[4], x[9], x[14]);
  }
  out[0] = x[0] + 0x61707865u; out[1] = x[1] + 0x3320646eu; out[2] = x[2] + 0x79622d32u; out[3] = x[3] + 0x6b206574u;
#pragma unroll
  for (int i = 0; i < 8; ++i) out[4 + i] = x[4 + i] + k[i];
  out[12] = x[12] + counter; out[13] = x[13] + n0; out[14] = x[14] + n1; out[15] = x[15] + n2;
}

// acc += sign * (block `counter` of the stream keyed k), sign < 0 subtracting (wrapping uint32 arithmetic)
COLEARN_HD void sa_add_block(uint32_t (&acc)[kSaWords], const uint32_t (&k)[8], int sign, uint32_t counter) {
  uint32_t w[kSaWords];
  sa_chacha20_block(k, counter, 0u, 0u, 0u, w);
#pragma unroll
  for (int i = 0; i < kSaWords; ++i) acc[i] += sign < 0 ? 0u - w[i] : w[i];
}

COLEARN_HD float sa_mul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}

COLEARN_HD float sa_div_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

// round to the nearest integer, ties to even (|x| < 2^31 here)
COLEARN_HD int32_t sa_f2i_rn(float x) {
#if defined(__CUDA_ARCH__)
  return __float2int_rn(x);
#else
  return (int32_t)rintf(x);
#endif
}

COLEARN_HD float sa_i2f_rn(int32_t z) {
#if defined(__CUDA_ARCH__)
  return __int2float_rn(z);
#else
  return (float)z;
#endif
}

// the fixed-point code of a delta d (clip > 0, scale = 2^f); counts the non-finite and the clipped deltas
COLEARN_HD uint32_t sa_encode(float d, float clip, float scale, int& clipped, int& nonfinite) {
  if (d != d) {
    ++nonfinite;
    return 0u;
  }
  const float a = fabsf(d);
  if (a == INFINITY) ++nonfinite;
  else if (a > clip) ++clipped;
  const float c = d > clip ? clip : (d < -clip ? -clip : d);
  return (uint32_t)sa_f2i_rn(sa_mul_rn(c, scale));
}

// the mean delta of n survivors whose codes sum to z (mod 2^32), inv_scale = 2^-f
COLEARN_HD float sa_decode(uint32_t z, float inv_scale, float n) {
  return sa_div_rn(sa_mul_rn(sa_i2f_rn((int32_t)z), inv_scale), n);
}

// Work split of the coordinator's correction streams.  0: fedavg_secagg_kernel expands every stream itself (enough ChaCha20
// columns to fill the GPU).  Otherwise a row too short for that (the FFNN has 151 columns) with many streams: secagg_streams_kernel
// first runs ceil(S / per) chunks of `per` streams per column and adds them into a uint32 scratch row with atomicAdd (wrapping
// addition is exact and commutative: the same bits in any order).
COLEARN_HD int sa_streams_per_task(int64_t n, int streams) {
  const int64_t cols = (n + kSaWords - 1) / kSaWords;
  const int64_t fill = 132 * 1024;                      // threads that keep an H100's 132 SMs busy
  if (cols >= 132 * 256 || streams <= 8) return 0;
  int64_t chunks = (streams + 3) / 4;                   // at least 4 streams per thread
  if (chunks > fill / cols) chunks = fill / cols;
  if (chunks <= 1) return 0;
  return (int)((streams + chunks - 1) / chunks);
}

}  // namespace colearn
