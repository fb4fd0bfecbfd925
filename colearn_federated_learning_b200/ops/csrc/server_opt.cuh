// Server optimizers of the FedOpt family (Reddi et al., "Adaptive Federated Optimization", ICLR 2021; server momentum:
// Hsu et al. 2019), applied per element inside the kernels that already form the FedAvg average a = sum_k w_k theta_k:
// star_round_kernel and twoshot_chunk (comm.cu), fedavg_opt_kernel (elementwise.cu).  This is the only definition of the
// arithmetic; the GPU build and the SIMT CPU build (host_shim.h) both compile it.  With d = a - theta:
//
//   sgd      theta += lr d                                          (kind 0: the kernels keep their own code for it)
//   avgm     m = b1 m + d                                           theta += lr m
//   adagrad  m = b1 m + (1 - b1) d ;  v = v + d^2                   theta += lr m / (sqrt(v) + tau)
//   adam     m = b1 m + (1 - b1) d ;  v = b2 v + (1 - b2) d^2       same
//   yogi     m = b1 m + (1 - b1) d ;  v = v - (1 - b2) d^2 sign(v - d^2)   same
//
// No bias correction (as in the paper).  m starts at 0 and v at tau^2.  IEEE sqrtf and division (the build does not use
// --use_fast_math).  Every product that could otherwise be contracted into an FMA on the GPU is written as an explicit fmaf,
// so that the GPU and the CPU build round the same way.
// Included by colearn_kernels.h after COLEARN_HD is defined.
#pragma once
#include <math.h>
#include <stdint.h>

namespace colearn {

enum ServerOptKind : int { SOPT_SGD = 0, SOPT_AVGM = 1, SOPT_ADAGRAD = 2, SOPT_ADAM = 3, SOPT_YOGI = 4 };

// Zero-initialised (memset) = kind 0 = plain FedAvg with the kernel's server_lr: every existing caller keeps its path.
struct ServerOptArgs {
  int kind;        // ServerOptKind
  float lr, beta1, beta2, tau;
  float* m;        // first moment, indexed like theta (local memory of the element's owner); every kind but sgd
  float* v;        // second moment (adagrad, adam, yogi)
};

// true when a launch with these arguments may run (kind 0 always may)
inline bool server_opt_args_ok(const ServerOptArgs& o) {
  if (o.kind == SOPT_SGD) return true;
  if (o.kind < SOPT_AVGM || o.kind > SOPT_YOGI || o.m == nullptr) return false;
  if (o.kind >= SOPT_ADAGRAD && o.v == nullptr) return false;
  return ((reinterpret_cast<uintptr_t>(o.m) | reinterpret_cast<uintptr_t>(o.v)) & 15) == 0;
}

// one element: returns the new theta, updates the moments in place
COLEARN_HD float server_opt_update(const ServerOptArgs& o, float theta, float avg, float& m, float& v) {
  const float d = avg - theta;
  if (o.kind == SOPT_SGD) return fmaf(o.lr, d, theta);
  if (o.kind == SOPT_AVGM) {
    m = fmaf(o.beta1, m, d);
    return fmaf(o.lr, m, theta);
  }
  m = fmaf(o.beta1, m, (1.f - o.beta1) * d);
  const float d2 = d * d;
  if (o.kind == SOPT_ADAGRAD) {
    v = fmaf(d, d, v);
  } else if (o.kind == SOPT_ADAM) {
    v = fmaf(o.beta2, v, (1.f - o.beta2) * d2);
  } else {
    const float s = (v > d2) ? 1.f : ((v < d2) ? -1.f : 0.f);
    v = fmaf(-(1.f - o.beta2) * s, d2, v);
  }
  return fmaf(o.lr, m / (sqrtf(v) + o.tau), theta);
}

// element i of the arena: moments read from / written back to o.m[i], o.v[i]
COLEARN_HD float server_opt_step(const ServerOptArgs& o, int64_t i, float theta, float avg) {
  const bool has_v = o.kind >= SOPT_ADAGRAD;
  float m = o.m[i], v = has_v ? o.v[i] : 0.f;
  theta = server_opt_update(o, theta, avg, m, v);
  o.m[i] = m;
  if (has_v) o.v[i] = v;
  return theta;
}

// elements 4 j4 .. 4 j4 + 3 (16-byte moment accesses)
COLEARN_HD float4 server_opt_step4(const ServerOptArgs& o, int64_t j4, float4 t, const float4& a) {
  const bool has_v = o.kind >= SOPT_ADAGRAD;
  float4 m = reinterpret_cast<const float4*>(o.m)[j4];
  float4 v = has_v ? reinterpret_cast<const float4*>(o.v)[j4] : make_float4(0.f, 0.f, 0.f, 0.f);
  t.x = server_opt_update(o, t.x, a.x, m.x, v.x);
  t.y = server_opt_update(o, t.y, a.y, m.y, v.y);
  t.z = server_opt_update(o, t.z, a.z, m.z, v.z);
  t.w = server_opt_update(o, t.w, a.w, m.w, v.w);
  reinterpret_cast<float4*>(o.m)[j4] = m;
  if (has_v) reinterpret_cast<float4*>(o.v)[j4] = v;
  return t;
}

}  // namespace colearn
