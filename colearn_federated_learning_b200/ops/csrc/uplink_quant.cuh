// Uplink compression of the client updates (QSGD / FedPAQ-style unbiased stochastic quantization): a client sends its delta
// d = theta_k - theta as int8 or int4 codes with one float32 scale per block of 256 elements, instead of its fp32 model.
// quantize_delta_kernel (encode) and fedavg_q_kernel / fedavg_q_robust_kernel (decode fused into the FedAvg apply) in
// elementwise.cu use these functions; the GPU build and the SIMT CPU build (host_shim.h) both compile them, and
// ops/reference.py encode_delta / decode_delta is the PyTorch transcription.
//
// Per block of kUqBlock consecutive elements (the last block may be partial), with L = 127 (int8) or 7 (int4):
//   s    = max |d_j| over the block (as the uint32 max of the bit patterns |d_j|: NaN and Inf sort above every finite value)
//   some d_j not finite             -> step = NaN (0x7fc00000), every q = 0
//   inv = L / s overflows (s == 0,  -> step = 0, every q = 0       (|d_j| <= s < L / FLT_MAX ~ 3.7e-37)
//     or s below L / FLT_MAX)
//   otherwise                       -> step = s / L, inv = L / s (IEEE float32 divisions)
//   u = d_j * inv, f = floorf(u), q = clamp(f + (r_j < u - f ? 1 : 0), -L, L)
//   r_j = (fmix32(key ^ (j * 0x9E3779B9)) >> 8) * 2^-24   (j: element index in the arena, wrapping uint32 arithmetic)
// Decode: d^_j = (float)q_j * step.  E[d^] = d up to float rounding and |d^ - d| <= step.  u is formed with __fmul_rn so that
// nvcc cannot contract d * inv - f into an FMA: every rounding is fixed, the GPU, the SIMT build and the reference agree bit
// for bit.  Decoding does not need the key.
// Included by colearn_kernels.h after COLEARN_HD is defined.
#pragma once
#include <float.h>
#include <stdint.h>
#include <string.h>

namespace colearn {

constexpr int kUqBlock = 256;

template <int BITS>
struct UqCodec {
  static_assert(BITS == 8 || BITS == 4, "int8 or int4 codes");
  static constexpr int kLevels = BITS == 8 ? 127 : 7;
  static constexpr int kBytesPerLane = BITS;   // 8 codes of one lane: 8 bytes (int8) or 4 bytes (int4)
};

// MurmurHash3 finalizer
COLEARN_HD uint32_t uq_fmix32(uint32_t h) {
  h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
  return h;
}

// r_j in [0, 1), a multiple of 2^-24: exact in float32
COLEARN_HD float uq_uniform(uint32_t key, uint32_t j) {
  return (float)(uq_fmix32(key ^ (j * 0x9E3779B9u)) >> 8) * 5.9604644775390625e-08f;
}

COLEARN_HD float uq_bits_to_float(uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __uint_as_float(b);
#else
  float f;
  memcpy(&f, &b, sizeof(f));
  return f;
#endif
}

COLEARN_HD uint32_t uq_abs_bits(float v) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(v) & 0x7fffffffu;
#else
  uint32_t b;
  memcpy(&b, &v, sizeof(b));
  return b & 0x7fffffffu;
#endif
}

// step (the block's wire scale) and inv from the uint32 max of |d_j| bit patterns; inv == 0 means "every q = 0"
COLEARN_HD void uq_block_scale(uint32_t smax_bits, int levels, float& step, float& inv) {
  if (smax_bits >= 0x7f800000u) {          // a NaN or an Inf in the block
    step = uq_bits_to_float(0x7fc00000u);
    inv = 0.f;
    return;
  }
  const float s = uq_bits_to_float(smax_bits);
  inv = (float)levels / s;
  if (!(inv <= FLT_MAX)) {                 // s == 0 (inv = +Inf) or L / s overflows
    step = 0.f;
    inv = 0.f;
    return;
  }
  step = s / (float)levels;
}

COLEARN_HD float uq_mul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}

// the code of element j (delta d) of a block with inverse scale inv (0: the block encodes as zeros)
COLEARN_HD int uq_encode(float d, float inv, uint32_t key, uint32_t j, int levels) {
  if (inv == 0.f) return 0;
  const float u = uq_mul_rn(d, inv);
  const float f = floorf(u);
  int q = (int)f + (uq_uniform(key, j) < u - f ? 1 : 0);
  q = q < -levels ? -levels : q;
  return q > levels ? levels : q;
}

COLEARN_HD float uq_decode(int q, float step) { return uq_mul_rn((float)q, step); }

// two's-complement nibble -> int
COLEARN_HD int uq_nibble(uint32_t packed, int i) { return (int)(packed << (28 - 4 * i)) >> 28; }

}  // namespace colearn
