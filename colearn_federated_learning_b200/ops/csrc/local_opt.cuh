// Local optimizer step of a device's fit (fl/local_opt.py): SGD with momentum / nesterov / weight decay, and Adam, one
// parameter at a time.  The definition follows torch.optim's single-tensor SGD and Adam in float32; ops/reference.py
// (local_opt_step) is the same sequence of operations in PyTorch, and the tests hold the two to the bit.  Shared by the
// optimizer instances of the persistent MLP kernel (mlp_persistent_opt.cu), their SIMT CPU build and the host executor
// (mlp_host.cpp), so it includes nothing and defines its own qualifiers.
//
// Every operation is written out as one correctly rounded float32 operation: on the GPU through the __f*_rn intrinsics,
// which nvcc never contracts into an FMA; on the CPU with contraction switched off inside these functions (GCC: the
// optimize attribute; clang: `#pragma clang fp contract(off)` in every body), so that a compiler targeting an FMA unit (an
// aarch64 device) cannot fuse them either.  GCC does not inline a function whose optimize attribute differs from its
// caller's, so a CPU loop over many elements calls local_opt_pass once and gets local_opt_elem inlined there.
//
// Per step t = 1, 2, ... of one fit (moments m, v start at 0; nothing is carried between fits):
//   g <- g + wd * theta                                            (skipped for wd = 0, as torch does)
//   SGD:  b <- g (t = 1),  b <- mu * b + g (t > 1);  d <- g + mu * b (nesterov) or b;  theta <- theta - lr * d
//         (mu = 0: no buffer, d = g)
//   Adam: m <- b1 * m + (1 - b1) * g;  v <- b2 * v + (1 - b2) * (g * g)
//         p1 <- p1 * b1, p2 <- p2 * b2 (running products from 1);  s = lr / (1 - p1), r = sqrt(1 - p2)
//         theta <- theta - (s * m) / (sqrt(v) / r + eps)
#pragma once

#if defined(__CUDACC__) && !defined(COLEARN_HOST_SHIM)
#define LOCAL_OPT_HD __host__ __device__ __forceinline__
#elif defined(__GNUC__) && !defined(__clang__)
#define LOCAL_OPT_HD inline __attribute__((optimize("fp-contract=off")))
#else
#define LOCAL_OPT_HD inline
#endif
#if defined(__clang__) && !defined(__CUDACC__)
#define LOCAL_OPT_NO_CONTRACT _Pragma("clang fp contract(off)")
#else
#define LOCAL_OPT_NO_CONTRACT
#endif

namespace colearn {

enum LocalOptKind : int { LOCAL_OPT_SGD = 1, LOCAL_OPT_ADAM = 2 };   // fl/local_opt.py KINDS

// Hyper-parameters of one fit's optimizer, checked by fl/local_opt.py before any launch.  SGD reads momentum, nesterov and
// weight_decay; Adam reads beta1, beta2, eps and weight_decay.
struct LocalOptArgs {
  int kind;
  int nesterov;
  float momentum;
  float weight_decay;
  float beta1;
  float beta2;
  float eps;
};

// What every thread forms once per step before the per-element pass.
struct LocalOptStep {
  int t;          // steps taken so far, this one included (1 on the first)
  float p1, p2;   // Adam: b1^t, b2^t as float32 running products
  float s;        // Adam: lr / (1 - p1)
  float r;        // Adam: sqrt(1 - p2)
};

#if defined(__CUDA_ARCH__)
#define LO_ADD(a, b) __fadd_rn(a, b)
#define LO_SUB(a, b) __fsub_rn(a, b)
#define LO_MUL(a, b) __fmul_rn(a, b)
#define LO_DIV(a, b) __fdiv_rn(a, b)
#define LO_SQRT(a) __fsqrt_rn(a)
#else
#define LO_ADD(a, b) ((a) + (b))
#define LO_SUB(a, b) ((a) - (b))
#define LO_MUL(a, b) ((a) * (b))
#define LO_DIV(a, b) ((a) / (b))
#define LO_SQRT(a) __builtin_sqrtf(a)
#endif

LOCAL_OPT_HD LocalOptStep local_opt_start() {
  LocalOptStep st;
  st.t = 0;
  st.p1 = 1.f;
  st.p2 = 1.f;
  st.s = 0.f;
  st.r = 1.f;
  return st;
}

// advance to the next step (call once per step, before its per-element pass)
LOCAL_OPT_HD void local_opt_next(LocalOptStep& st, const LocalOptArgs& a, float lr) {
  LOCAL_OPT_NO_CONTRACT
  st.t += 1;
  if (a.kind == LOCAL_OPT_ADAM) {
    st.p1 = LO_MUL(st.p1, a.beta1);
    st.p2 = LO_MUL(st.p2, a.beta2);
    st.s = LO_DIV(lr, LO_SUB(1.f, st.p1));
    st.r = LO_SQRT(LO_SUB(1.f, st.p2));
  }
}

// one element: theta and its moments m (SGD: the momentum buffer) and v (Adam only) updated in place from its gradient g
LOCAL_OPT_HD void local_opt_elem(const LocalOptArgs& a, const LocalOptStep& st, float lr, float& theta, float g, float& m,
                                 float& v) {
  LOCAL_OPT_NO_CONTRACT
  if (a.weight_decay != 0.f) g = LO_ADD(g, LO_MUL(a.weight_decay, theta));
  if (a.kind == LOCAL_OPT_ADAM) {
    m = LO_ADD(LO_MUL(a.beta1, m), LO_MUL(LO_SUB(1.f, a.beta1), g));
    v = LO_ADD(LO_MUL(a.beta2, v), LO_MUL(LO_SUB(1.f, a.beta2), LO_MUL(g, g)));
    theta = LO_SUB(theta, LO_DIV(LO_MUL(st.s, m), LO_ADD(LO_DIV(LO_SQRT(v), st.r), a.eps)));
  } else {
    float d = g;   // momentum 0: no buffer, as torch.optim.SGD
    if (a.momentum != 0.f) {
      m = st.t == 1 ? g : LO_ADD(LO_MUL(a.momentum, m), g);
      d = a.nesterov ? LO_ADD(g, LO_MUL(a.momentum, m)) : m;
    }
    theta = LO_SUB(theta, LO_MUL(lr, d));
  }
}

// one step over n elements on the CPU (the host executor, tests): local_opt_next, then local_opt_elem for every element
LOCAL_OPT_HD void local_opt_pass(const LocalOptArgs& a, LocalOptStep& st, float lr, float* theta, const float* g, float* m,
                                 float* v, long long n) {
  LOCAL_OPT_NO_CONTRACT
  local_opt_next(st, a, lr);
  for (long long i = 0; i < n; ++i) local_opt_elem(a, st, lr, theta[i], g[i], m[i], v[i]);
}

#undef LO_ADD
#undef LO_SUB
#undef LO_MUL
#undef LO_DIV
#undef LO_SQRT

}  // namespace colearn
