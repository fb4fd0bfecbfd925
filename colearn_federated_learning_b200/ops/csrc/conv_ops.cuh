// Per-work-item bodies of the NHWC convolution / BatchNorm / pooling kernels (SURVEY K17).
//
// Every kernel in convnet.cu is either a *map* (one independent work item per loop iteration) or a *two-phase
// block* (phase 1 fills shared memory, __syncthreads, phase 2 drains it).  The bodies live here as
// host+device functions so that the exact same index arithmetic can be run on the CPU
// (conv_emul.cpp, built with g++ for the CPU test-suite) — the authoring box has no GPU.
//
// Layout: activations are NHWC flattened to a row-major matrix [M = N*H*W, C] of bf16; a convolution is
//   im2col (k = (kh, kw, c), so 8 consecutive k are 8 consecutive channels = one 16-byte load)
//   -> wgmma GEMM    z[M, Cout] = col[M, K] * Wp[Cout, K]^T        (gemm_wgmma.cu)
//   -> BatchNorm statistics / apply (+ residual, + ReLU).
// Backward: BatchNorm backward -> dgrad GEMM dcol = dz * (Wp^T)^T -> col2im gather (no atomics), and the
// wgrad GEMM dz^T * col^T with the SGD step fused in its epilogue.
#pragma once
#include <cuda_bf16.h>
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define CL_HD __host__ __device__ __forceinline__
#else
#define CL_HD inline
#endif
// L2-coherent load (skips L1): used where one CTA reads what other CTAs of the same launch just wrote
#if defined(__CUDA_ARCH__)
#define CL_LD_CG(p) __ldcg(p)
#else
#define CL_LD_CG(p) (*(p))
#endif

namespace colearn {
namespace convops {

struct alignas(16) BF8 {
  __nv_bfloat16 v[8];
};

CL_HD float bf2f(__nv_bfloat16 x) { return __bfloat162float(x); }
CL_HD __nv_bfloat16 f2bf(float x) { return __float2bfloat16(x); }

// ------------------------------------------------------------------------------------------------------
// im2col: col[m, k] = x[n, oh*stride - pad + kh, ow*stride - pad + kw, c],  k = (kh*KW + kw)*C + c,
// zero outside the image and for k in [K, K_pad).  x is addressed through element strides so the stem can
// read the user's NCHW fp32 batch directly.
// ------------------------------------------------------------------------------------------------------
struct Im2colArgs {
  const void* x;
  int x_f32;                    // 1: x is float, 0: bf16
  int vec;                      // 1: C % 8 == 0, sC == 1, bf16, 16-byte aligned rows -> 128-bit loads
  long long sN, sH, sW, sC;     // element strides of x
  int N, H, W, C, KH, KW, stride, pad, OH, OW;
  int K;                        // KH*KW*C
  int K_pad;                    // pitch of col (multiple of 8)
  __nv_bfloat16* col;           // [N*OH*OW, K_pad]
};
CL_HD long long im2col_items(const Im2colArgs& a) { return (long long)a.N * a.OH * a.OW * (a.K_pad / 8); }
CL_HD void im2col_body(const Im2colArgs& a, long long item) {
  const int kg = a.K_pad / 8;
  const long long m = item / kg;
  const int k0 = (int)(item % kg) * 8;
  const int ow = (int)(m % a.OW);
  const int oh = (int)((m / a.OW) % a.OH);
  const int n = (int)(m / ((long long)a.OW * a.OH));
  BF8 out;
  if (a.vec && k0 < a.K) {
    const int c0 = k0 % a.C, kk = k0 / a.C;
    const int kw = kk % a.KW, kh = kk / a.KW;
    const int ih = oh * a.stride - a.pad + kh, iw = ow * a.stride - a.pad + kw;
    if (ih >= 0 && ih < a.H && iw >= 0 && iw < a.W) {
      const __nv_bfloat16* src = reinterpret_cast<const __nv_bfloat16*>(a.x) + n * a.sN + ih * a.sH + iw * a.sW + c0;
      out = *reinterpret_cast<const BF8*>(src);
    } else {
      for (int j = 0; j < 8; ++j) out.v[j] = f2bf(0.f);
    }
  } else {
    for (int j = 0; j < 8; ++j) {
      const int k = k0 + j;
      float v = 0.f;
      if (k < a.K) {
        const int c = k % a.C, kk = k / a.C;
        const int kw = kk % a.KW, kh = kk / a.KW;
        const int ih = oh * a.stride - a.pad + kh, iw = ow * a.stride - a.pad + kw;
        if (ih >= 0 && ih < a.H && iw >= 0 && iw < a.W) {
          const long long off = n * a.sN + ih * a.sH + iw * a.sW + c * a.sC;
          v = a.x_f32 ? reinterpret_cast<const float*>(a.x)[off] : bf2f(reinterpret_cast<const __nv_bfloat16*>(a.x)[off]);
        }
      }
      out.v[j] = f2bf(v);
    }
  }
  *reinterpret_cast<BF8*>(a.col + m * a.K_pad + k0) = out;
}

// ------------------------------------------------------------------------------------------------------
// col2im as a gather (the adjoint of im2col without atomics):
//   dx[n,h,w,c] = add[n,h,w,c] + sum_{kh,kw} dcol[(n,oh,ow), (kh*KW+kw)*C + c]   with oh*stride - pad + kh == h
// ------------------------------------------------------------------------------------------------------
struct Col2imArgs {
  const __nv_bfloat16* dcol;    // [N*OH*OW, K_pad]
  int K_pad;
  int N, H, W, C, KH, KW, stride, pad, OH, OW;   // C % 8 == 0
  const __nv_bfloat16* add;     // optional [N*H*W, C]
  __nv_bfloat16* dx;            // [N*H*W, C]
};
CL_HD long long col2im_items(const Col2imArgs& a) { return (long long)a.N * a.H * a.W * (a.C / 8); }
CL_HD void col2im_body(const Col2imArgs& a, long long item) {
  const int cg = a.C / 8;
  const long long mi = item / cg;
  const int c0 = (int)(item % cg) * 8;
  const int w = (int)(mi % a.W);
  const int h = (int)((mi / a.W) % a.H);
  const int n = (int)(mi / ((long long)a.W * a.H));
  float acc[8];
  if (a.add) {
    const BF8 t = *reinterpret_cast<const BF8*>(a.add + mi * a.C + c0);
    for (int j = 0; j < 8; ++j) acc[j] = bf2f(t.v[j]);
  } else {
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  }
  for (int kh = 0; kh < a.KH; ++kh) {
    const int th = h + a.pad - kh;
    if (th < 0 || th % a.stride != 0) continue;
    const int oh = th / a.stride;
    if (oh >= a.OH) continue;
    for (int kw = 0; kw < a.KW; ++kw) {
      const int tw = w + a.pad - kw;
      if (tw < 0 || tw % a.stride != 0) continue;
      const int ow = tw / a.stride;
      if (ow >= a.OW) continue;
      const long long mo = ((long long)n * a.OH + oh) * a.OW + ow;
      const BF8 t = *reinterpret_cast<const BF8*>(a.dcol + mo * a.K_pad + (kh * a.KW + kw) * a.C + c0);
      for (int j = 0; j < 8; ++j) acc[j] += bf2f(t.v[j]);
    }
  }
  BF8 o;
  for (int j = 0; j < 8; ++j) o.v[j] = f2bf(acc[j]);
  *reinterpret_cast<BF8*>(a.dx + mi * a.C + c0) = o;
}

// ------------------------------------------------------------------------------------------------------
// BatchNorm reductions (two-phase block: 256 threads = 32 row lanes x 8 column groups of 8 channels, i.e. a
// block owns 64 channels x rows_per_block rows and emits one partial per channel and quantity).
//   mode 0 (forward statistics): q1 = x,  q2 = x^2
//   mode 1 (backward):           q1 = g,  q2 = g * xhat,   g = dy * (out > 0 if out != null),  xhat = (x-mean)*invstd
// partial is [nseg, 2, C] fp32; bn_finalize_body reduces it.
// ------------------------------------------------------------------------------------------------------
constexpr int kBnLanes = 32;          // row lanes per block
constexpr int kBnCols = 64;           // channels per block
constexpr int kBnThreads = 256;
constexpr int kBnSmemFloats = 2 * kBnLanes * kBnCols;

struct BnReduceArgs {
  int mode;
  const __nv_bfloat16* x;       // [M, ldx] conv output (pre-normalisation); channels [0, C) are used
  int ldx;
  const __nv_bfloat16* dy;      // [M, C] (mode 1)
  const __nv_bfloat16* out;     // [M, C] post-activation output for the ReLU mask, or null (mode 1)
  const float* mean;            // [C] (mode 1)
  const float* invstd;          // [C] (mode 1)
  int M, C;                     // C % 64 == 0
  int rows_per_block;
  float* partial;               // [nseg, 2, C]
};
CL_HD int bn_nseg(const BnReduceArgs& a) { return (a.M + a.rows_per_block - 1) / a.rows_per_block; }
CL_HD void bn_reduce_phase1(const BnReduceArgs& a, int bx, int by, int tid, float* smem) {
  const int cg = tid % 8, rl = tid / 8;
  const int c0 = bx * kBnCols + cg * 8;
  const int r_end = (by + 1) * a.rows_per_block < a.M ? (by + 1) * a.rows_per_block : a.M;
  float s1[8], s2[8], mu[8], is[8];
  for (int j = 0; j < 8; ++j) {
    s1[j] = 0.f; s2[j] = 0.f; mu[j] = 0.f; is[j] = 1.f;
  }
  if (a.mode == 1) {
    for (int j = 0; j < 8; ++j) {
      mu[j] = a.mean[c0 + j];
      is[j] = a.invstd[c0 + j];
    }
  }
  for (int r = by * a.rows_per_block + rl; r < r_end; r += kBnLanes) {
    const BF8 xv = *reinterpret_cast<const BF8*>(a.x + (long long)r * a.ldx + c0);
    if (a.mode == 0) {
      for (int j = 0; j < 8; ++j) {
        const float v = bf2f(xv.v[j]);
        s1[j] += v;
        s2[j] += v * v;
      }
    } else {
      const BF8 dv = *reinterpret_cast<const BF8*>(a.dy + (long long)r * a.C + c0);
      BF8 ov;
      if (a.out) ov = *reinterpret_cast<const BF8*>(a.out + (long long)r * a.C + c0);
      for (int j = 0; j < 8; ++j) {
        float g = bf2f(dv.v[j]);
        if (a.out && !(bf2f(ov.v[j]) > 0.f)) g = 0.f;
        const float xh = (bf2f(xv.v[j]) - mu[j]) * is[j];
        s1[j] += g;
        s2[j] += g * xh;
      }
    }
  }
  for (int j = 0; j < 8; ++j) {
    smem[(0 * kBnLanes + rl) * kBnCols + cg * 8 + j] = s1[j];
    smem[(1 * kBnLanes + rl) * kBnCols + cg * 8 + j] = s2[j];
  }
}
CL_HD void bn_reduce_phase2(const BnReduceArgs& a, int bx, int by, int tid, const float* smem) {
  if (tid >= 2 * kBnCols) return;
  const int q = tid / kBnCols, c = tid % kBnCols;
  float s = 0.f;
  for (int rl = 0; rl < kBnLanes; ++rl) s += smem[(q * kBnLanes + rl) * kBnCols + c];
  a.partial[((long long)by * 2 + q) * a.C + bx * kBnCols + c] = s;
}

struct BnFinalizeArgs {
  int mode;                     // 0: statistics, 1: parameter gradients
  const float* partial;         // [nseg, 2, C]
  int nseg, M, C;
  float eps, momentum;
  float* mean;                  // mode 0 outputs
  float* invstd;
  float* running_mean;          // optional, updated in place (torch semantics: unbiased variance)
  float* running_var;
  float* dgamma;                // mode 1 outputs
  float* dbeta;
};
template <bool kCoherent = false>
CL_HD void bn_finalize_body(const BnFinalizeArgs& a, int c) {
  double s1 = 0.0, s2 = 0.0;
  for (int s = 0; s < a.nseg; ++s) {
    const float* p1 = a.partial + ((long long)s * 2 + 0) * a.C + c;
    const float* p2 = a.partial + ((long long)s * 2 + 1) * a.C + c;
    s1 += (double)(kCoherent ? CL_LD_CG(p1) : *p1);
    s2 += (double)(kCoherent ? CL_LD_CG(p2) : *p2);
  }
  if (a.mode == 0) {
    const double mean = s1 / a.M;
    double var = s2 / a.M - mean * mean;
    if (var < 0.0) var = 0.0;
    a.mean[c] = (float)mean;
    a.invstd[c] = (float)(1.0 / sqrt(var + (double)a.eps));
    if (a.running_mean) {
      const double unbiased = a.M > 1 ? var * a.M / (a.M - 1) : var;
      a.running_mean[c] = (float)((1.0 - a.momentum) * a.running_mean[c] + a.momentum * mean);
      a.running_var[c] = (float)((1.0 - a.momentum) * a.running_var[c] + a.momentum * unbiased);
    }
  } else {
    a.dbeta[c] = (float)s1;
    a.dgamma[c] = (float)s2;
  }
}

// Reduction + finalize in ONE launch: every block bumps a per-column-group counter after publishing its partial;
// the block that observes the last ticket finalises that group's 64 channels (threadfence-reduction pattern) and
// resets the counter, so the buffer is reusable without a memset.
struct BnFusedArgs {
  BnReduceArgs r;
  BnFinalizeArgs f;
  unsigned int* counters;       // [C / 64], zero before the first use
};
CL_HD void bn_fused_phase3(const BnFusedArgs& a, int bx, int tid) {
  if (tid < kBnCols) bn_finalize_body<true>(a.f, bx * kBnCols + tid);
}

// out = relu?( (x - mean) * invstd * gamma + beta (+ res) )
struct BnApplyArgs {
  const __nv_bfloat16* x;       // [M, ldx]
  int ldx;
  const float* mean;
  const float* invstd;
  const float* gamma;
  const float* beta;
  const __nv_bfloat16* res;     // optional [M, C]
  int relu;
  int M, C;                     // C % 8 == 0
  __nv_bfloat16* out;           // [M, C]
};
CL_HD long long bn_apply_items(const BnApplyArgs& a) { return (long long)a.M * (a.C / 8); }
CL_HD void bn_apply_body(const BnApplyArgs& a, long long item) {
  const int cg = a.C / 8;
  const long long r = item / cg;
  const int c0 = (int)(item % cg) * 8;
  const BF8 xv = *reinterpret_cast<const BF8*>(a.x + r * a.ldx + c0);
  BF8 rv, o;
  if (a.res) rv = *reinterpret_cast<const BF8*>(a.res + r * a.C + c0);
  for (int j = 0; j < 8; ++j) {
    const int c = c0 + j;
    float y = (bf2f(xv.v[j]) - a.mean[c]) * a.invstd[c] * a.gamma[c] + a.beta[c];
    if (a.res) y += bf2f(rv.v[j]);
    if (a.relu && !(y > 0.f)) y = 0.f;
    o.v[j] = f2bf(y);
  }
  *reinterpret_cast<BF8*>(a.out + r * a.C + c0) = o;
}

// dx = gamma * invstd * (g - dbeta/M - xhat * dgamma/M),  g = dy * (out > 0 if out != null); optionally emits g
struct BnBwdArgs {
  const __nv_bfloat16* x;       // [M, ldx]
  int ldx;
  const __nv_bfloat16* dy;      // [M, C]
  const __nv_bfloat16* out;     // optional ReLU mask source
  const float* mean;
  const float* invstd;
  const float* gamma;
  const float* dgamma;
  const float* dbeta;
  int M, C;
  __nv_bfloat16* dx;            // [M, C]
  __nv_bfloat16* g_out;         // optional [M, C]: the masked upstream gradient (identity branch of a residual block)
};
CL_HD long long bn_bwd_items(const BnBwdArgs& a) { return (long long)a.M * (a.C / 8); }
CL_HD void bn_bwd_body(const BnBwdArgs& a, long long item) {
  const int cg = a.C / 8;
  const long long r = item / cg;
  const int c0 = (int)(item % cg) * 8;
  const BF8 xv = *reinterpret_cast<const BF8*>(a.x + r * a.ldx + c0);
  const BF8 dv = *reinterpret_cast<const BF8*>(a.dy + r * a.C + c0);
  BF8 ov, o, go;
  if (a.out) ov = *reinterpret_cast<const BF8*>(a.out + r * a.C + c0);
  const float inv_m = 1.f / (float)a.M;
  for (int j = 0; j < 8; ++j) {
    const int c = c0 + j;
    float g = bf2f(dv.v[j]);
    if (a.out && !(bf2f(ov.v[j]) > 0.f)) g = 0.f;
    const float xh = (bf2f(xv.v[j]) - a.mean[c]) * a.invstd[c];
    o.v[j] = f2bf(a.gamma[c] * a.invstd[c] * (g - a.dbeta[c] * inv_m - xh * a.dgamma[c] * inv_m));
    go.v[j] = f2bf(g);
  }
  *reinterpret_cast<BF8*>(a.dx + r * a.C + c0) = o;
  if (a.g_out) *reinterpret_cast<BF8*>(a.g_out + r * a.C + c0) = go;
}

// ------------------------------------------------------------------------------------------------------
// Max pooling (padding behaves as -inf, first maximum wins — torch semantics) and its gather backward.
// ------------------------------------------------------------------------------------------------------
struct PoolArgs {
  const __nv_bfloat16* x;       // fwd: [N*H*W, C] input        bwd: unused
  __nv_bfloat16* out;           // fwd: [N*OH*OW, C] output     bwd: dx [N*H*W, C]
  unsigned char* idx;           // [N*OH*OW, C] window offset kh*KW+kw of the maximum (fwd: written, bwd: read)
  const __nv_bfloat16* dy;      // bwd: [N*OH*OW, C]
  int N, H, W, C, KH, KW, stride, pad, OH, OW;
};
CL_HD long long maxpool_fwd_items(const PoolArgs& a) { return (long long)a.N * a.OH * a.OW * (a.C / 8); }
CL_HD void maxpool_fwd_body(const PoolArgs& a, long long item) {
  const int cg = a.C / 8;
  const long long mo = item / cg;
  const int c0 = (int)(item % cg) * 8;
  const int ow = (int)(mo % a.OW);
  const int oh = (int)((mo / a.OW) % a.OH);
  const int n = (int)(mo / ((long long)a.OW * a.OH));
  float best[8];
  int arg[8];
  bool have = false;
  for (int j = 0; j < 8; ++j) {
    best[j] = 0.f;
    arg[j] = 0;
  }
  for (int kh = 0; kh < a.KH; ++kh) {
    const int ih = oh * a.stride - a.pad + kh;
    if (ih < 0 || ih >= a.H) continue;
    for (int kw = 0; kw < a.KW; ++kw) {
      const int iw = ow * a.stride - a.pad + kw;
      if (iw < 0 || iw >= a.W) continue;
      const BF8 t = *reinterpret_cast<const BF8*>(a.x + (((long long)n * a.H + ih) * a.W + iw) * a.C + c0);
      for (int j = 0; j < 8; ++j) {
        const float v = bf2f(t.v[j]);
        if (!have || v > best[j]) {
          best[j] = v;
          arg[j] = kh * a.KW + kw;
        }
      }
      have = true;
    }
  }
  BF8 o;
  for (int j = 0; j < 8; ++j) {
    o.v[j] = f2bf(best[j]);
    a.idx[mo * a.C + c0 + j] = (unsigned char)arg[j];
  }
  *reinterpret_cast<BF8*>(a.out + mo * a.C + c0) = o;
}
CL_HD long long maxpool_bwd_items(const PoolArgs& a) { return (long long)a.N * a.H * a.W * (a.C / 8); }
CL_HD void maxpool_bwd_body(const PoolArgs& a, long long item) {
  const int cg = a.C / 8;
  const long long mi = item / cg;
  const int c0 = (int)(item % cg) * 8;
  const int w = (int)(mi % a.W);
  const int h = (int)((mi / a.W) % a.H);
  const int n = (int)(mi / ((long long)a.W * a.H));
  float acc[8];
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int kh = 0; kh < a.KH; ++kh) {
    const int th = h + a.pad - kh;
    if (th < 0 || th % a.stride != 0) continue;
    const int oh = th / a.stride;
    if (oh >= a.OH) continue;
    for (int kw = 0; kw < a.KW; ++kw) {
      const int tw = w + a.pad - kw;
      if (tw < 0 || tw % a.stride != 0) continue;
      const int ow = tw / a.stride;
      if (ow >= a.OW) continue;
      const long long mo = ((long long)n * a.OH + oh) * a.OW + ow;
      const BF8 t = *reinterpret_cast<const BF8*>(a.dy + mo * a.C + c0);
      const int code = kh * a.KW + kw;
      for (int j = 0; j < 8; ++j)
        if (a.idx[mo * a.C + c0 + j] == code) acc[j] += bf2f(t.v[j]);
    }
  }
  BF8 o;
  for (int j = 0; j < 8; ++j) o.v[j] = f2bf(acc[j]);
  *reinterpret_cast<BF8*>(a.out + mi * a.C + c0) = o;
}

// Global average pooling [N, HW, C] -> [N, C] and its backward (dx = dy / HW broadcast).
struct AvgPoolArgs {
  const __nv_bfloat16* in;      // fwd: x [N*HW, C]   bwd: dy [N, C]
  __nv_bfloat16* out;           // fwd: [N, C]         bwd: dx [N*HW, C]
  int N, HW, C;
};
CL_HD long long avgpool_fwd_items(const AvgPoolArgs& a) { return (long long)a.N * (a.C / 8); }
CL_HD void avgpool_fwd_body(const AvgPoolArgs& a, long long item) {
  const int cg = a.C / 8;
  const long long n = item / cg;
  const int c0 = (int)(item % cg) * 8;
  float acc[8];
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int p = 0; p < a.HW; ++p) {
    const BF8 t = *reinterpret_cast<const BF8*>(a.in + (n * a.HW + p) * a.C + c0);
    for (int j = 0; j < 8; ++j) acc[j] += bf2f(t.v[j]);
  }
  BF8 o;
  const float inv = 1.f / (float)a.HW;
  for (int j = 0; j < 8; ++j) o.v[j] = f2bf(acc[j] * inv);
  *reinterpret_cast<BF8*>(a.out + n * a.C + c0) = o;
}
CL_HD long long avgpool_bwd_items(const AvgPoolArgs& a) { return (long long)a.N * a.HW * (a.C / 8); }
CL_HD void avgpool_bwd_body(const AvgPoolArgs& a, long long item) {
  const int cg = a.C / 8;
  const long long mi = item / cg;
  const int c0 = (int)(item % cg) * 8;
  const long long n = mi / a.HW;
  const BF8 t = *reinterpret_cast<const BF8*>(a.in + n * a.C + c0);
  BF8 o;
  const float inv = 1.f / (float)a.HW;
  for (int j = 0; j < 8; ++j) o.v[j] = f2bf(bf2f(t.v[j]) * inv);
  *reinterpret_cast<BF8*>(a.out + mi * a.C + c0) = o;
}

// ------------------------------------------------------------------------------------------------------
// Weight packing.  torch keeps a conv weight as [Cout, Cin, KH, KW]; the GEMMs want [Cout_pad, K_pad] with
// k = (kh*KW + kw)*Cin + c, zero padded to tile multiples.  During a local fit the *packed* fp32 copy is the
// master the wgrad epilogue updates; pack (arena -> packed fp32 + bf16) runs once before, unpack once after.
// One launch handles every layer through a descriptor table.
// ------------------------------------------------------------------------------------------------------
struct PackDesc {
  long long src_off;            // element offset of the [rows, cols] matrix in the flat arena
  long long dst_off;            // element offset of the [rows_pad, cols_pad] matrix in the packed buffers
  int rows, cols, rows_pad, cols_pad;
  int C;                        // channels for the (c, kh, kw) -> (kh, kw, c) permutation; 0 = plain matrix
  int KHW;                      // KH*KW
};
struct PackArgs {
  float* arena;                 // flat fp32 arena (state-dict order)
  float* packed_f32;            // [total]
  __nv_bfloat16* packed_bf16;   // [total] or null
  const PackDesc* descs;
  int n_desc;
  long long total;              // sum rows_pad*cols_pad
  int unpack;                   // 0: arena -> packed (+bf16);  1: packed_f32 -> arena
};
CL_HD void pack_body(const PackArgs& a, long long e) {
  int d = 0, hi = a.n_desc - 1;   // last descriptor with dst_off <= e
  while (d < hi) {
    const int mid = (d + hi + 1) / 2;
    if (a.descs[mid].dst_off <= e) d = mid; else hi = mid - 1;
  }
  const PackDesc& L = a.descs[d];
  const long long loc = e - L.dst_off;
  const int r = (int)(loc / L.cols_pad), k = (int)(loc % L.cols_pad);
  const bool valid = r < L.rows && k < L.cols;
  long long src = 0;
  if (valid) {
    int col = k;
    if (L.C > 0) {
      const int c = k % L.C, kk = k / L.C;
      col = c * L.KHW + kk;
    }
    src = L.src_off + (long long)r * L.cols + col;
  }
  if (a.unpack) {
    if (valid) a.arena[src] = a.packed_f32[e];
  } else {
    const float v = valid ? a.arena[src] : 0.f;
    a.packed_f32[e] = v;
    if (a.packed_bf16) a.packed_bf16[e] = f2bf(v);
  }
}

// ------------------------------------------------------------------------------------------------------
// Work decomposition of the persistent wgmma GEMM (gemm_wgmma.cu).  Every role of a CTA (TMA producer, consumer
// warpgroups) walks the same list: work unit w = blockIdx.x, blockIdx.x + gridDim.x, ...;  w / S is the output tile,
// w % S the K slice (S = split_k, 1 = off).  Host+device so that the CPU test-suite can check that the units tile the
// output exactly once and that the slices partition K.
// L2-friendly rasterisation: the tiles are walked in groups of kGroupM m-units x all n-blocks (m fastest inside a group),
// so that the CTAs running concurrently share a small set of A row-slabs and B column-slabs (an 8192^3 GEMM has 134 MB
// of A alone; the naive order streams all of it once per n-block).
// ------------------------------------------------------------------------------------------------------
constexpr int kGroupM = 8;
CL_HD void work_to_tile(int w, int m_units, int n_tiles, int& m_unit, int& n_blk) {
  const int group_size = kGroupM * n_tiles;
  const int group_id = w / group_size;
  const int first_m = group_id * kGroupM;
  const int gsz = (m_units - first_m) < kGroupM ? (m_units - first_m) : kGroupM;
  const int r = w - group_id * group_size;
  m_unit = first_m + (r % gsz);
  n_blk = r / gsz;
}
// k-block range of K slice s of S: [split_kb(s), split_kb(s + 1)); non-empty for every s when num_kb >= S
CL_HD int split_kb(int num_kb, int s, int S) { return (int)(((long long)num_kb * s) / S); }

// ------------------------------------------------------------------------------------------------------
// Implicit GEMM addressing (stride-1 convolutions on NHWC activations whose images are <= 128 pixels).
// The activation [N, H, W, C] is described to TMA as a 4-D tensor (c, w, h, n); a GEMM tile of 128 (or 64) pixels is a
// box of whole images (c: 64, w: W, h: H, n: pixels / (H*W)), and tap (kh, kw) of the filter is the same box moved by
// (kw - pad, kh - pad): what falls outside the image is zero-filled by TMA — the convolution's padding.  The box lands
// in shared memory as [pixels x 64 channels] lines of 128 bytes, i.e. exactly the operand tile the explicit im2col
// GEMM reads, so no col matrix exists.  One decode serves the three GEMMs of a convolution:
//   forward (mode 1, flip 0):  A = x boxes,  K = (tap, c):   z[p, co]  = sum x[p + tap - pad, c]  * Wp[co, tap*C + c]
//   dgrad   (mode 1, flip 1):  A = dz boxes, K = (tap, co):  dx[p, c]  = sum dz[p + pad - tap, co] * Wt[tap*Cin + c, co]
//   wgrad   (mode 2):          B = x boxes (MN-major), reduction over pixels:
//                                                           dW[co, tap*C + c] = sum_p dz[p, co] * x[p + tap - pad, c]
// ------------------------------------------------------------------------------------------------------
struct ConvAddr {
  int mode;        // 0: off   1: the A operand is an activation (K-major boxes of 128 pixels)   2: the B operand is (MN-major, 64 pixels)
  int flip;        // mode 1: 0 = forward (coordinate tap - pad), 1 = dgrad (pad - tap)
  int C;           // channels of the activation behind the 4-D map (multiple of 64)
  int KH, KW, pad;
  int HW;          // H*W of the activation: 1, 4, 16 or 64 (whole images per box)
  int n_images;    // N (a fully padded K/N block is pushed out of bounds with this)
  int b_rows_per_tap;  // mode 1 / flip 1: rows of W^T per tap (= Cin of the convolution = N of the GEMM)
  int b_mn;        // mode 1 / flip 1: the weight operand is the packed Wp[co, (tap, ci)] itself (MN-major B) instead of W^T
  int tap_lo;      // mode 1: first filter tap of the K loop and ...
  int tap_cnt;     // ... how many (0 = all KH*KW).  1x1 images only ever see the centre tap — every other tap's box lies
                   // entirely in the padding — so the launcher walks that one tap (K = C instead of KH*KW*C)
};
struct ConvBox {
  int c, w, h, n;  // 4-D TMA coordinates of the activation box
  int b_col, b_row;  // mode 1: 2-D coordinates of the weight box (column = k offset, row = first output column)
};
// mode 1: k-block kb (64 channels of one tap) of the output tile starting at pixel m0 / output column n0
CL_HD ConvBox conv_kblock(const ConvAddr& g, int kb, int m0, int n0) {
  const int cblocks = g.C / 64;
  const int tap = g.tap_lo + kb / cblocks, cb = kb % cblocks;
  const int kh = tap / g.KW, kw = tap % g.KW;
  ConvBox b;
  b.c = cb * 64;
  b.w = g.flip ? g.pad - kw : kw - g.pad;
  b.h = g.flip ? g.pad - kh : kh - g.pad;
  b.n = m0 / g.HW;
  if (g.flip) {
    b.b_col = cb * 64;                          // K index inside W^T's row = output channel of the convolution
    b.b_row = tap * g.b_rows_per_tap + n0;
  } else {
    b.b_col = tap * g.C + cb * 64;              // k = tap*C + c, the packed weights' own column order
    b.b_row = n0;
  }
  return b;
}
// mode 2: the 64-column block `blk` (= k / 64, k = tap*C + c) of the B operand for the reduction block kb (64 pixels);
// blocks past the last tap (the K padding of the packed weights) are placed out of bounds = zeros
CL_HD ConvBox conv_nblock(const ConvAddr& g, int blk, int kb) {
  const int cblocks = g.C / 64;
  const int tap = blk / cblocks, cb = blk % cblocks;
  const int kh = tap / g.KW, kw = tap % g.KW;
  ConvBox b;
  b.c = cb * 64;
  b.w = kw - g.pad;
  b.h = kh - g.pad;
  b.n = tap < g.KH * g.KW ? (kb * 64) / g.HW : g.n_images;
  b.b_col = 0;
  b.b_row = 0;
  return b;
}

// ------------------------------------------------------------------------------------------------------
// Split-K reduction: the wgmma GEMM in split-K mode leaves S raw fp32 partial accumulators part[s, rows, cols]
// (gemm_wgmma.cu, GemmEpilogue::split_k); this map sums them in slice order (deterministic) and applies the
// epilogue the un-split GEMM would have fused:
//   master != null : fused SGD of the wgrad GEMMs  master -= lr * sum ; shadow = bf16(master)
//   else           : out_bf16 = bf16(sum)          (conv forward: the next activation matrix)
// One work item = 4 consecutive elements (float4 loads, one 8-byte bf16x4 store).
// ------------------------------------------------------------------------------------------------------
struct alignas(8) BF4 {
  __nv_bfloat16 v[4];
};
struct alignas(16) F4 {
  float v[4];
};
struct SplitKReduceArgs {
  const float* part;            // [S, numel]
  int S;
  long long numel;              // rows * cols of one slice (multiple of 4)
  float* master;                // [numel] fp32 master weights, updated in place; or null
  float lr;
  __nv_bfloat16* shadow;        // [numel] bf16 copy of the updated master; or null
  __nv_bfloat16* out_bf16;      // [numel] bf16(sum) when master == null
};
CL_HD long long splitk_reduce_items(const SplitKReduceArgs& a) { return a.numel / 4; }
CL_HD void splitk_reduce_body(const SplitKReduceArgs& a, long long item) {
  const long long e = item * 4;
  F4 acc = *reinterpret_cast<const F4*>(a.part + e);
  for (int s = 1; s < a.S; ++s) {
    const F4 t = *reinterpret_cast<const F4*>(a.part + (long long)s * a.numel + e);
    for (int j = 0; j < 4; ++j) acc.v[j] += t.v[j];
  }
  BF4 o;
  if (a.master) {
    F4 w = *reinterpret_cast<const F4*>(a.master + e);
    for (int j = 0; j < 4; ++j) w.v[j] = fmaf(-a.lr, acc.v[j], w.v[j]);   // same expression as the fused GEMM epilogue
    *reinterpret_cast<F4*>(a.master + e) = w;
    if (!a.shadow) return;
    for (int j = 0; j < 4; ++j) o.v[j] = f2bf(w.v[j]);
    *reinterpret_cast<BF4*>(a.shadow + e) = o;
  } else {
    for (int j = 0; j < 4; ++j) o.v[j] = f2bf(acc.v[j]);
    *reinterpret_cast<BF4*>(a.out_bf16 + e) = o;
  }
}

}  // namespace convops
}  // namespace colearn
