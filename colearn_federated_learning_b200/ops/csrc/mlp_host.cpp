// Host (CPU) executor of the worker-side local fit for the MLP family — the native path of devices WITHOUT a GPU.
//
// The reference's workers are Raspberry Pis running PySyft's FederatedClient._fit in Python/torch (SURVEY C27:
// 163.7 batch-1 SGD steps/s on an RPi 3B+, BASELINE.md); this repo's remote_worker.py on a CPU-only device, the
// coordinator's VirtualWorker mode on a CPU-only box (BASELINE config 1) and the gloo test engine used to run the
// PyTorch definitions in ops/reference.py (~200 us per step of op-dispatch overhead for a 5 k-MAC network).  This file
// is the same fit — shuffled batches, forward, loss, backward, SGD, max_nr_batches — as one C++ loop on the flat fp32
// arena, with K clients trained concurrently on K threads (the GIL is released).  Semantics are those of
// ops/reference.py::mlp_local_sgd / loss_and_dz (tests compare the two); the sm_90a persistent kernel
// (mlp_persistent.cu) is the GPU counterpart.  Built with g++ only (ops/build.py::build_host), links the CPU libtorch.
#include <torch/extension.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include "local_opt.cuh"

namespace py = pybind11;

namespace {

enum Loss : int { BCE = 0, SSE = 1, XENT = 2, MSE = 3 };   // = LossKind in colearn_kernels.h / fused_mlp.LOSS_CODES

struct Net {
  std::vector<int> dims;         // d_in, hidden..., d_out
  std::vector<int64_t> w_off;    // offset of W_l [dims[l+1], dims[l]] in the flat arena (state-dict order: W, b, W, b...)
  std::vector<int64_t> b_off;
  int64_t n_params = 0;
  int max_dim = 0;
  bool sigmoid_out = false;
  explicit Net(const std::vector<int64_t>& d, bool sig) : sigmoid_out(sig) {
    TORCH_CHECK(d.size() >= 2, "dims needs at least an input and an output size");
    for (int64_t v : d) {
      TORCH_CHECK(v > 0 && v < (1 << 20), "bad layer size");
      dims.push_back((int)v);
      max_dim = std::max(max_dim, (int)v);
    }
    for (size_t l = 0; l + 1 < dims.size(); ++l) {
      w_off.push_back(n_params);
      n_params += (int64_t)dims[l] * dims[l + 1];
      b_off.push_back(n_params);
      n_params += dims[l + 1];
    }
  }
  int layers() const { return (int)dims.size() - 1; }
};

struct Task {
  const float* x = nullptr;      // [n, d_in]
  const float* y = nullptr;      // [n, y_dim]
  const int* perm = nullptr;     // [perm_rows, n] or null (identity)
  float* theta = nullptr;        // [n_params], trained in place
  int n = 0, y_dim = 1, perm_rows = 1;
  float last = 0.f, mean = 0.f;  // results
  int steps = 0;
};

struct Hyper {
  int batch, epochs, max_steps, loss;
  float lr;
  const float* cw = nullptr;   // a class-weighted fit: w[class of the row] (its label y[0]) scales the row's loss and gradient
  const colearn::LocalOptArgs* opt = nullptr;   // a local optimizer (local_opt.cuh) instead of plain SGD: the generic loop only
};

// Per-thread scratch: activations of every layer for every sample of the batch, dz ping-pong, gradient arena (B > 1)
struct Scratch {
  std::vector<float> acts;       // [layers + 1][B][max_dim]
  std::vector<float> dz, dprev;  // [max_dim]
  std::vector<float> grad;       // [n_params] (used when B > 1 or with a local optimizer)
  std::vector<float> m, v;       // [n_params] the local optimizer's moments (this fit's)
  std::vector<float> dout;       // [B][d_out]: dL/d(pre-activation of the last layer)
};

inline float clamp_log(float v) { return v < -100.f ? -100.f : v; }

// forward of one sample; a[l] = input of layer l (a[0] = x), a[L] = network output (post output-activation)
__attribute__((always_inline)) inline void forward_one(const Net& net, const float* theta, const float* x, float* acts, int stride_l) {
  const int L = net.layers();
  std::memcpy(acts, x, sizeof(float) * net.dims[0]);
  for (int l = 0; l < L; ++l) {
    const int k = net.dims[l], n = net.dims[l + 1];
    const float* w = theta + net.w_off[l];
    const float* b = theta + net.b_off[l];
    const float* in = acts + (int64_t)l * stride_l;
    float* out = acts + (int64_t)(l + 1) * stride_l;
    for (int j = 0; j < n; ++j) {
      const float* wr = w + (int64_t)j * k;
      float s = 0.f;
#pragma omp simd reduction(+ : s)
      for (int i = 0; i < k; ++i) s += wr[i] * in[i];
      s += b[j];
      if (l < L - 1) s = s <= 0.f ? 0.f : s;   // ReLU that keeps NaN, like torch.relu
      else if (net.sigmoid_out) s = 1.f / (1.f + std::exp(-s));
      out[j] = s;
    }
  }
}

// loss value of the batch and dL/d(pre-activation of the last layer) per sample (ops/reference.py::loss_and_dz); cw: class
// weights (nullptr: none)
__attribute__((always_inline)) inline float loss_and_dout(const Net& net, int loss, const float* acts, int stride_b, int stride_l, const float* const* ys, int y_dim,
                           int bsz, float* dout, const float* cw) {
  const int L = net.layers(), d = net.dims[L];
  double value = 0.0;
  for (int s = 0; s < bsz; ++s) {
    const float* out = acts + (int64_t)s * stride_b + (int64_t)L * stride_l;
    float* dz = dout + (int64_t)s * d;
    const float* y = ys[s];
    const float r = cw ? cw[(int)y[0]] : 1.f;
    if (loss == XENT) {
      const int label = (int)y[0];
      float mx = out[0];
      for (int j = 1; j < d; ++j) mx = std::max(mx, out[j]);
      float se = 0.f;
      for (int j = 0; j < d; ++j) se += std::exp(out[j] - mx);
      const float lse = mx + std::log(se);
      const float term = lse - out[label >= 0 && label < d ? label : 0];
      value += (double)(cw ? r * term : term);
      for (int j = 0; j < d; ++j) {
        const float g = (std::exp(out[j] - lse) - (j == label ? 1.f : 0.f)) / (float)bsz;
        dz[j] = cw ? g * r : g;
      }
    } else if (loss == BCE) {
      const float inv0 = 1.f / (float)(bsz * d), inv = cw ? inv0 * r : inv0;
      for (int j = 0; j < d; ++j) {
        const float p = out[j], t = y_dim >= d ? y[j] : y[0];
        value -= (double)(t * clamp_log(std::log(p)) + (1.f - t) * clamp_log(std::log1p(-p))) * inv;
        dz[j] = (p - t) * inv;
      }
    } else {   // SSE / MSE
      const float scale0 = loss == SSE ? 1.f : 1.f / (float)bsz, scale = cw ? scale0 * r : scale0;
      for (int j = 0; j < d; ++j) {
        const float diff = out[j] - (y_dim >= d ? y[j] : y[0]);
        value += (double)(diff * diff * scale);
        float g = 2.f * diff * scale;
        if (net.sigmoid_out) g *= out[j] * (1.f - out[j]);
        dz[j] = g;
      }
    }
  }
  if (loss == XENT) value /= bsz;
  return (float)value;
}

// Function multi-versioning: the same loop compiled for AVX2+FMA (x86-64-v3) next to the portable baseline; the loader
// picks the best clone for the CPU it runs on (the in-tree .so travels between boxes, so no -march=native).
#if defined(__x86_64__) && defined(__GNUC__) && !defined(__clang__)
#define COLEARN_CLONES __attribute__((target_clones("arch=x86-64-v3", "default")))
#else
#define COLEARN_CLONES
#endif

COLEARN_CLONES
void run_fit(const Net& net, Task& t, const Hyper& hp, Scratch& sc) {
  const int L = net.layers(), B = hp.batch, md = net.max_dim;
  const int stride_l = md, stride_b = (L + 1) * md;
  sc.acts.assign((size_t)B * stride_b, 0.f);
  sc.dz.assign(md, 0.f);
  sc.dprev.assign(md, 0.f);
  sc.dout.assign((size_t)B * net.dims[L], 0.f);
  const bool acc = B > 1 || hp.opt != nullptr;   // accumulate the batch gradient, then step
  if (acc) sc.grad.assign((size_t)net.n_params, 0.f);
  colearn::LocalOptStep ost = colearn::local_opt_start();
  if (hp.opt != nullptr) {
    sc.m.assign((size_t)net.n_params, 0.f);
    sc.v.assign((size_t)net.n_params, 0.f);
  }
  std::vector<const float*> ys(B);
  float* theta = t.theta;
  double loss_sum = 0.0;
  int it = 0;
  bool done = false;
  for (int e = 0; e < hp.epochs && !done; ++e) {
    const int* order = t.perm ? t.perm + (int64_t)(e % t.perm_rows) * t.n : nullptr;
    for (int lo = 0; lo < t.n && !done; lo += B) {
      const int bsz = std::min(B, t.n - lo);
      for (int s = 0; s < bsz; ++s) {
        const int idx = order ? order[lo + s] : lo + s;
        forward_one(net, theta, t.x + (int64_t)idx * net.dims[0], sc.acts.data() + (int64_t)s * stride_b, stride_l);
        ys[s] = t.y + (int64_t)idx * t.y_dim;
      }
      t.last = loss_and_dout(net, hp.loss, sc.acts.data(), stride_b, stride_l, ys.data(), t.y_dim, bsz, sc.dout.data(), hp.cw);
      loss_sum += t.last;
      if (acc) std::fill(sc.grad.begin(), sc.grad.end(), 0.f);
      for (int s = 0; s < bsz; ++s) {
        const float* acts = sc.acts.data() + (int64_t)s * stride_b;
        std::memcpy(sc.dz.data(), sc.dout.data() + (int64_t)s * net.dims[L], sizeof(float) * net.dims[L]);
        for (int l = L - 1; l >= 0; --l) {
          const int k = net.dims[l], n = net.dims[l + 1];
          float* w = theta + net.w_off[l];
          float* b = theta + net.b_off[l];
          const float* a = acts + (int64_t)l * stride_l;
          const float* dz = sc.dz.data();
          if (l > 0) {   // dz_{l-1} = (W^T dz) * relu'(a) with the weights of BEFORE this step
            float* dp = sc.dprev.data();
            for (int i = 0; i < k; ++i) dp[i] = 0.f;
            for (int j = 0; j < n; ++j) {
              const float g = dz[j];
              const float* wr = w + (int64_t)j * k;
              for (int i = 0; i < k; ++i) dp[i] += g * wr[i];
            }
            for (int i = 0; i < k; ++i)
              if (a[i] <= 0.f) dp[i] = 0.f;   // threshold_backward: a NaN activation passes the gradient
          }
          if (!acc) {   // batch-1 plain SGD (the reference's Arguments): apply the update right away, no gradient arena
            for (int j = 0; j < n; ++j) {
              const float g = hp.lr * dz[j];
              float* wr = w + (int64_t)j * k;
              for (int i = 0; i < k; ++i) wr[i] -= g * a[i];
              b[j] -= g;
            }
          } else {
            float* gw = sc.grad.data() + net.w_off[l];
            float* gb = sc.grad.data() + net.b_off[l];
            for (int j = 0; j < n; ++j) {
              const float g = dz[j];
              float* gr = gw + (int64_t)j * k;
              for (int i = 0; i < k; ++i) gr[i] += g * a[i];
              gb[j] += g;
            }
          }
          if (l > 0) std::swap(sc.dz, sc.dprev);
        }
      }
      if (hp.opt != nullptr) {
        const float* g = sc.grad.data();
        colearn::local_opt_pass(*hp.opt, ost, hp.lr, theta, g, sc.m.data(), sc.v.data(), net.n_params);
      } else if (B > 1) {
        const float* g = sc.grad.data();
        for (int64_t i = 0; i < net.n_params; ++i) theta[i] -= hp.lr * g[i];
      }
      ++it;
      if (hp.max_steps > 0 && it >= hp.max_steps) done = true;
    }
  }
  t.steps = it;
  t.mean = it > 0 ? (float)(loss_sum / it) : 0.f;
}

// ---- fixed-shape fast path (batch 1) --------------------------------------------------------------------------------------
// The reference's three networks have compile-time layer widths: with constant trip counts the compiler unrolls and
// vectorises every dot product / AXPY exactly (no remainder loops, no alignment peeling — which is most of the time for
// 10- to 64-element loops): 1.33 -> 0.69 us per step for the 10-64-64-2 net, 0.99 -> 0.51 for the FFNN on the authoring box.
// Same operations as run_fit (batch 1); only the association inside a dot product follows the vector width the compiler
// picks, so the two paths agree to rounding (1e-7 against the PyTorch reference after 600 steps), not bit for bit.
// COLEARN_HOST_GENERIC=1 forces the generic loop.
template <int... D>
struct Shape {
  static constexpr int L = sizeof...(D) - 1;
  static constexpr int dims[sizeof...(D)] = {D...};
  static constexpr int max_dim() { int m = 0; for (int d : dims) m = d > m ? d : m; return m; }
  static constexpr int w_off(int l) { int o = 0; for (int i = 0; i < l; ++i) o += dims[i] * dims[i + 1] + dims[i + 1]; return o; }
  static constexpr int b_off(int l) { return w_off(l) + dims[l] * dims[l + 1]; }
  static bool matches(const Net& net) {
    if (net.layers() != L) return false;
    for (int i = 0; i <= L; ++i) if (net.dims[i] != dims[i]) return false;
    return true;
  }
};

template <class S, int l>
__attribute__((always_inline)) inline void fixed_forward(const float* theta, float (*acts)[S::max_dim()], bool sigmoid_out) {
  if constexpr (l < S::L) {
    constexpr int K = S::dims[l], N = S::dims[l + 1];
    const float* w = theta + S::w_off(l);
    const float* b = theta + S::b_off(l);
    const float* in = acts[l];
    float* out = acts[l + 1];
    for (int j = 0; j < N; ++j) {
      const float* wr = w + j * K;
      float s = 0.f;
#pragma omp simd reduction(+ : s)
      for (int i = 0; i < K; ++i) s += wr[i] * in[i];
      s += b[j];
      if (l < S::L - 1) s = s <= 0.f ? 0.f : s;   // (keeps NaN)
      else if (sigmoid_out) s = 1.f / (1.f + std::exp(-s));
      out[j] = s;
    }
    fixed_forward<S, l + 1>(theta, acts, sigmoid_out);
  }
}

template <class S, int l>
__attribute__((always_inline)) inline void fixed_backward(float* theta, const float (*acts)[S::max_dim()], float* dz, float* dprev, float lr) {
  if constexpr (l >= 0) {
    constexpr int K = S::dims[l], N = S::dims[l + 1];
    float* w = theta + S::w_off(l);
    float* b = theta + S::b_off(l);
    const float* a = acts[l];
    if constexpr (l > 0) {   // dz_{l-1} = (W^T dz) * relu'(a) with the weights of BEFORE this step
      for (int i = 0; i < K; ++i) dprev[i] = 0.f;
      for (int j = 0; j < N; ++j) {
        const float g = dz[j];
        const float* wr = w + j * K;
#pragma omp simd
        for (int i = 0; i < K; ++i) dprev[i] += g * wr[i];
      }
      for (int i = 0; i < K; ++i)
        if (a[i] <= 0.f) dprev[i] = 0.f;
    }
    for (int j = 0; j < N; ++j) {
      const float g = lr * dz[j];
      float* wr = w + j * K;
#pragma omp simd
      for (int i = 0; i < K; ++i) wr[i] -= g * a[i];
      b[j] -= g;
    }
    if constexpr (l > 0) fixed_backward<S, l - 1>(theta, acts, dprev, dz, lr);   // dz / dprev swap roles
  }
}

template <class S>
COLEARN_CLONES void run_fit_fixed(const Net& net, Task& t, const Hyper& hp, Scratch& sc) {
  constexpr int MD = S::max_dim(), L = S::L;
  alignas(64) float acts[L + 1][MD];
  alignas(64) float dz[MD], dprev[MD];
  sc.dout.assign((size_t)net.dims[L], 0.f);
  float* theta = t.theta;
  double loss_sum = 0.0;
  int it = 0;
  bool done = false;
  for (int e = 0; e < hp.epochs && !done; ++e) {
    const int* order = t.perm ? t.perm + (int64_t)(e % t.perm_rows) * t.n : nullptr;
    for (int lo = 0; lo < t.n && !done; ++lo) {
      const int idx = order ? order[lo] : lo;
      std::memcpy(acts[0], t.x + (int64_t)idx * S::dims[0], sizeof(float) * S::dims[0]);
      fixed_forward<S, 0>(theta, acts, net.sigmoid_out);
      const float* y = t.y + (int64_t)idx * t.y_dim;
      t.last = loss_and_dout(net, hp.loss, &acts[0][0], (L + 1) * MD, MD, &y, t.y_dim, 1, sc.dout.data(), hp.cw);
      loss_sum += t.last;
      std::memcpy(dz, sc.dout.data(), sizeof(float) * S::dims[L]);
      fixed_backward<S, L - 1>(theta, acts, dz, dprev, hp.lr);
      ++it;
      if (hp.max_steps > 0 && it >= hp.max_steps) done = true;
    }
  }
  t.steps = it;
  t.mean = it > 0 ? (float)(loss_sum / it) : 0.f;
}

using ShapeMLP64 = Shape<10, 64, 64, 2>;         // BASELINE MLP
using ShapeFFNN = Shape<10, 50, 30, 10, 1>;      // the reference's FFNN (cf.py:22-44)
using ShapeTestingRemote = Shape<2, 50, 10, 1>;  // the reference's TestingRemote (cf.py:46-55)

// one local fit: the fixed-shape path for the known networks at batch-1 plain SGD, the generic loop otherwise
inline void run_fit_any(const Net& net, Task& t, const Hyper& hp, Scratch& sc) {
  static const bool generic_only = std::getenv("COLEARN_HOST_GENERIC") != nullptr;
  if (hp.batch == 1 && hp.opt == nullptr && !generic_only) {
    if (ShapeMLP64::matches(net)) return run_fit_fixed<ShapeMLP64>(net, t, hp, sc);
    if (ShapeFFNN::matches(net)) return run_fit_fixed<ShapeFFNN>(net, t, hp, sc);
    if (ShapeTestingRemote::matches(net)) return run_fit_fixed<ShapeTestingRemote>(net, t, hp, sc);
  }
  run_fit(net, t, hp, sc);
}

Task make_task(const Net& net, const torch::Tensor& theta, const torch::Tensor& x, const torch::Tensor& y,
               const c10::optional<torch::Tensor>& perm) {
  auto ok = [](const torch::Tensor& t, at::ScalarType st) { return !t.is_cuda() && t.scalar_type() == st && t.is_contiguous(); };
  TORCH_CHECK(ok(theta, at::kFloat) && theta.dim() == 1 && theta.numel() == net.n_params, "theta: contiguous CPU fp32 [", net.n_params, "]");
  TORCH_CHECK(ok(x, at::kFloat) && x.dim() == 2 && x.size(1) == net.dims[0], "x: contiguous CPU fp32 [n, ", net.dims[0], "]");
  TORCH_CHECK(ok(y, at::kFloat) && y.dim() == 2 && y.size(0) == x.size(0), "y: contiguous CPU fp32 [n, y_dim]");
  Task t;
  t.x = x.data_ptr<float>();
  t.y = y.data_ptr<float>();
  t.theta = theta.data_ptr<float>();
  t.n = (int)x.size(0);
  t.y_dim = (int)y.size(1);
  if (perm.has_value()) {
    TORCH_CHECK(ok(*perm, at::kInt) && perm->dim() == 2 && perm->size(1) == x.size(0) && perm->size(0) >= 1, "perm: contiguous CPU int32 [rows, n]");
    t.perm = perm->data_ptr<int>();
    t.perm_rows = (int)perm->size(0);
    const int* p = t.perm;
    for (int64_t i = 0; i < perm->numel(); ++i) TORCH_CHECK(p[i] >= 0 && p[i] < t.n, "perm entry out of range");
  }
  return t;
}

// K clients, each trained in place on its own arena, min(K, threads) at a time.  Returns [K, 2] = {last, mean} losses.
// class_weights (mlp_local_sgd_cw): one weight per class; every row's label y[0] must be a class index below their count.
torch::Tensor fit_host(std::vector<int64_t> dims, bool sigmoid_out, std::vector<torch::Tensor> thetas,
                       std::vector<torch::Tensor> xs, std::vector<torch::Tensor> ys,
                       std::vector<c10::optional<torch::Tensor>> perms, int64_t batch_size, int64_t epochs,
                       int64_t max_nr_batches, int64_t loss, double lr, int64_t threads, const std::vector<double>* class_weights,
                       const std::vector<double>* local_opt = nullptr) {
  const Net net(dims, sigmoid_out);
  const size_t K = thetas.size();
  TORCH_CHECK(K >= 1 && xs.size() == K && ys.size() == K && perms.size() == K, "one theta / x / y / perm per client");
  TORCH_CHECK(batch_size >= 1 && epochs >= 0 && loss >= 0 && loss <= 3, "bad hyper-parameters");
  TORCH_CHECK(loss != BCE || sigmoid_out, "bce needs a sigmoid head");
  std::vector<Task> tasks;
  for (size_t i = 0; i < K; ++i) {
    tasks.push_back(make_task(net, thetas[i], xs[i], ys[i], perms[i]));
    if (loss == XENT) TORCH_CHECK(tasks.back().y_dim >= 1, "xent needs a label column");
  }
  std::vector<float> cw;
  if (class_weights != nullptr) {
    for (double w : *class_weights) cw.push_back((float)w);
    TORCH_CHECK(!cw.empty(), "no class weights");
    for (const Task& t : tasks)
      for (int i = 0; i < t.n; ++i) {
        const float c = t.y[(int64_t)i * t.y_dim];
        TORCH_CHECK(c >= 0.f && c < (float)cw.size() && c == (float)(int)c, "label of row ", i, " is not a class index below ", cw.size());
      }
  }
  colearn::LocalOptArgs lo{};
  if (local_opt != nullptr) {
    TORCH_CHECK(local_opt->size() == 7, "local optimizer: 7 values");
    const std::vector<double>& o = *local_opt;
    lo = colearn::LocalOptArgs{(int)o[0], (int)o[1], (float)o[2], (float)o[3], (float)o[4], (float)o[5], (float)o[6]};
    TORCH_CHECK(lo.kind == colearn::LOCAL_OPT_SGD || lo.kind == colearn::LOCAL_OPT_ADAM, "unknown local optimizer kind");
  }
  const Hyper hp{(int)batch_size, (int)epochs, (int)max_nr_batches, (int)loss, (float)lr, class_weights ? cw.data() : nullptr,
                 local_opt ? &lo : nullptr};
  int nthreads = threads > 0 ? (int)threads : (int)std::thread::hardware_concurrency();
  nthreads = std::max(1, std::min<int>(nthreads, (int)K));
  {
    py::gil_scoped_release nogil;
    if (nthreads == 1) {
      Scratch sc;
      for (auto& t : tasks) run_fit_any(net, t, hp, sc);
    } else {
      std::vector<std::thread> pool;
      for (int w = 0; w < nthreads; ++w)
        pool.emplace_back([&, w] {
          Scratch sc;
          for (size_t i = w; i < K; i += nthreads) run_fit_any(net, tasks[i], hp, sc);
        });
      for (auto& th : pool) th.join();
    }
  }
  auto out = torch::zeros({(int64_t)K, 2}, torch::kFloat);
  float* o = out.data_ptr<float>();
  for (size_t i = 0; i < K; ++i) {
    o[2 * i] = tasks[i].last;
    o[2 * i + 1] = tasks[i].mean;
  }
  return out;
}
torch::Tensor mlp_local_sgd_host(std::vector<int64_t> dims, bool sigmoid_out, std::vector<torch::Tensor> thetas,
                                 std::vector<torch::Tensor> xs, std::vector<torch::Tensor> ys,
                                 std::vector<c10::optional<torch::Tensor>> perms, int64_t batch_size, int64_t epochs,
                                 int64_t max_nr_batches, int64_t loss, double lr, int64_t threads) {
  return fit_host(dims, sigmoid_out, thetas, xs, ys, perms, batch_size, epochs, max_nr_batches, loss, lr, threads, nullptr);
}
torch::Tensor mlp_local_sgd_cw_host(std::vector<int64_t> dims, bool sigmoid_out, std::vector<torch::Tensor> thetas,
                                    std::vector<torch::Tensor> xs, std::vector<torch::Tensor> ys,
                                    std::vector<c10::optional<torch::Tensor>> perms, int64_t batch_size, int64_t epochs,
                                    int64_t max_nr_batches, int64_t loss, double lr, int64_t threads, std::vector<double> class_weights) {
  return fit_host(dims, sigmoid_out, thetas, xs, ys, perms, batch_size, epochs, max_nr_batches, loss, lr, threads, &class_weights);
}
// the generic loop with a local optimizer's step (local_opt.cuh); local_opt: {kind, nesterov, momentum, weight_decay, beta1,
// beta2, eps}, checked by the caller (fl/local_opt.py)
torch::Tensor mlp_local_sgd_opt_host(std::vector<int64_t> dims, bool sigmoid_out, std::vector<torch::Tensor> thetas,
                                     std::vector<torch::Tensor> xs, std::vector<torch::Tensor> ys,
                                     std::vector<c10::optional<torch::Tensor>> perms, int64_t batch_size, int64_t epochs,
                                     int64_t max_nr_batches, int64_t loss, double lr, int64_t threads, std::vector<double> local_opt) {
  return fit_host(dims, sigmoid_out, thetas, xs, ys, perms, batch_size, epochs, max_nr_batches, loss, lr, threads, nullptr, &local_opt);
}

// Batched forward (inference / evaluation): out [n, d_out], post output-activation
torch::Tensor mlp_forward_host(std::vector<int64_t> dims, bool sigmoid_out, torch::Tensor theta, torch::Tensor x) {
  const Net net(dims, sigmoid_out);
  TORCH_CHECK(!theta.is_cuda() && theta.scalar_type() == at::kFloat && theta.is_contiguous() && theta.numel() == net.n_params, "theta");
  TORCH_CHECK(!x.is_cuda() && x.scalar_type() == at::kFloat && x.is_contiguous() && x.dim() == 2 && x.size(1) == net.dims[0], "x");
  const int64_t n = x.size(0);
  const int L = net.layers(), d = net.dims[L];
  auto out = torch::empty({n, (int64_t)d}, torch::kFloat);
  std::vector<float> acts((size_t)(L + 1) * net.max_dim);
  const float* th = theta.data_ptr<float>();
  const float* xp = x.data_ptr<float>();
  float* op = out.data_ptr<float>();
  for (int64_t i = 0; i < n; ++i) {
    forward_one(net, th, xp + i * net.dims[0], acts.data(), net.max_dim);
    std::memcpy(op + i * d, acts.data() + (int64_t)L * net.max_dim, sizeof(float) * d);
  }
  return out;
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "colearn host executor: MLP local SGD / forward on CPU devices (no CUDA dependency)";
  m.def("mlp_local_sgd", &mlp_local_sgd_host);
  m.def("mlp_local_sgd_cw", &mlp_local_sgd_cw_host);
  m.def("mlp_local_sgd_opt", &mlp_local_sgd_opt_host);
  m.def("mlp_forward", &mlp_forward_host);
}
