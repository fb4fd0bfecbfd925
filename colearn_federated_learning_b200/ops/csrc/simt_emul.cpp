// Python face of the SIMT-on-CPU build: mlp_persistent.cu (+ mlp_v2.cuh), elementwise.cu and comm.cu — the kernel
// sources themselves — are compiled with g++ through host_shim.h (simt_mlp.cpp / simt_elementwise.cpp / simt_comm.cpp,
// one OS thread per CUDA thread) and driven here through the same launch_* entry points bindings.cpp uses on a GPU.
// Tests only (ops/build.py::build_simt_emul, tests/test_simt_emul.py).
#define COLEARN_HOST_SHIM 1
#include <torch/extension.h>

#include "colearn_kernels.h"

namespace py = pybind11;

namespace {
using torch::Tensor;

const float* fptr(const Tensor& t, const char* name) {
  TORCH_CHECK(!t.is_cuda() && t.scalar_type() == at::kFloat && t.is_contiguous(), name, ": contiguous CPU fp32");
  return t.data_ptr<float>();
}

// K clients (one emulated CTA each, run one after the other).  theta_outs[i] may alias theta_in.
// Returns losses [K, 2] = {last, mean}; flags (int32 [K], optional) receive signal_value = 7 + i.
// class_weights (mlp_local_sgd_cw): the class-weighted instances of mlp_persistent_cw.cu; nullptr: the unweighted ones.
Tensor mlp_fit(int64_t net_kind, Tensor theta_in, std::vector<Tensor> theta_outs, std::vector<Tensor> xs, std::vector<Tensor> ys,
               std::vector<c10::optional<Tensor>> perms, int64_t batch_size, int64_t epochs, int64_t max_steps, int64_t loss,
               double lr, int64_t variant, std::vector<double> out_scales, bool delta_mode, c10::optional<Tensor> flags,
               int64_t perm_seed, int64_t perm_row0, c10::optional<Tensor> perm_scratch, const std::vector<double>* class_weights,
               const std::vector<double>* local_opt = nullptr) {
  const size_t K = xs.size();
  TORCH_CHECK(K >= 1 && ys.size() == K && perms.size() == K && theta_outs.size() == K && out_scales.size() == K, "one entry per client");
  const int P = colearn::mlp_net_num_params((int)net_kind);
  TORCH_CHECK(P > 0 && theta_in.numel() == P, "theta_in must hold ", P, " parameters");
  Tensor losses = torch::zeros({(int64_t)K, 2}, torch::kFloat);
  std::vector<colearn::ClientDesc> descs(K);
  for (size_t i = 0; i < K; ++i) {
    colearn::ClientDesc& d = descs[i];
    memset(&d, 0, sizeof(d));
    d.x = fptr(xs[i], "x");
    d.y = fptr(ys[i], "y");
    TORCH_CHECK(xs[i].dim() == 2 && ys[i].dim() == 2 && xs[i].size(0) == ys[i].size(0), "x [n, d_in], y [n, y_dim]");
    d.n = (int)xs[i].size(0);
    d.y_dim = (int)ys[i].size(1);
    d.perm_rows = 1;
    if (perms[i].has_value()) {
      const Tensor& p = *perms[i];
      TORCH_CHECK(!p.is_cuda() && p.scalar_type() == at::kInt && p.is_contiguous() && p.dim() == 2 && p.size(1) == d.n, "perm int32 [rows, n]");
      d.perm = p.data_ptr<int>();
      d.perm_rows = (int)p.size(0);
    } else if (perm_seed != 0) {                                   // in-kernel shuffle (ClientDesc::perm_seed): client i keys on seed + i
      d.perm_seed = (uint64_t)(perm_seed + (int64_t)i);
      d.perm_row0 = (int)perm_row0;
      if (perm_scratch.has_value()) {
        TORCH_CHECK(perm_scratch->scalar_type() == at::kInt && perm_scratch->is_contiguous() && perm_scratch->dim() == 2 &&
                    perm_scratch->size(0) == (int64_t)K && perm_scratch->size(1) >= epochs * (int64_t)d.n, "perm_scratch int32 [K, epochs * n]");
        d.perm_scratch = perm_scratch->data_ptr<int>() + (int64_t)i * perm_scratch->size(1);
      }
    }
    d.theta_in = fptr(theta_in, "theta_in");
    TORCH_CHECK(theta_outs[i].numel() == P, "theta_out size");
    d.theta_out = const_cast<float*>(fptr(theta_outs[i], "theta_out"));
    d.loss_out = losses.data_ptr<float>() + 2 * i;
    d.out_scale = (float)out_scales[i];
    d.delta_mode = delta_mode ? 1 : 0;
    if (flags.has_value()) {
      TORCH_CHECK(flags->scalar_type() == at::kInt && flags->is_contiguous() && flags->numel() >= (int64_t)K, "flags int32 [K]");
      d.signal_flag = reinterpret_cast<uint32_t*>(flags->data_ptr<int>()) + i;
      d.signal_value = 7u + (uint32_t)i;
    }
  }
  colearn::SgdHyper hp;
  hp.batch_size = (int)batch_size;
  hp.epochs = (int)epochs;
  hp.max_steps = (int)max_steps;
  hp.loss = (int)loss;
  hp.lr = (float)lr;
  hp.variant = (int)variant;
  {
    py::gil_scoped_release nogil;
    cudaError_t e;
    if (local_opt != nullptr) {
      TORCH_CHECK(local_opt->size() == 7, "local optimizer: 7 values");
      const std::vector<double>& o = *local_opt;
      const colearn::LocalOptArgs lo{(int)o[0], (int)o[1], (float)o[2], (float)o[3], (float)o[4], (float)o[5], (float)o[6]};
      e = colearn::launch_mlp_local_sgd_opt((int)net_kind, descs.data(), (int)K, hp, lo, nullptr);
    } else if (class_weights != nullptr) {
      colearn::ClassWeights cw{};
      TORCH_CHECK(class_weights->size() <= 8, "at most 8 class weights");
      for (size_t c = 0; c < class_weights->size(); ++c) cw.w[c] = (float)(*class_weights)[c];
      e = colearn::launch_mlp_local_sgd_cw((int)net_kind, descs.data(), (int)K, hp, cw, nullptr);
    } else {
      e = colearn::launch_mlp_local_sgd((int)net_kind, descs.data(), (int)K, hp, nullptr);
    }
    TORCH_CHECK(e == cudaSuccess, "launch_mlp_local_sgd (host shim) failed");
  }
  return losses;
}
Tensor mlp_local_sgd(int64_t net_kind, Tensor theta_in, std::vector<Tensor> theta_outs, std::vector<Tensor> xs, std::vector<Tensor> ys,
                     std::vector<c10::optional<Tensor>> perms, int64_t batch_size, int64_t epochs, int64_t max_steps, int64_t loss,
                     double lr, int64_t variant, std::vector<double> out_scales, bool delta_mode, c10::optional<Tensor> flags,
                     int64_t perm_seed, int64_t perm_row0, c10::optional<Tensor> perm_scratch) {
  return mlp_fit(net_kind, theta_in, theta_outs, xs, ys, perms, batch_size, epochs, max_steps, loss, lr, variant, out_scales, delta_mode,
                 flags, perm_seed, perm_row0, perm_scratch, nullptr);
}
Tensor mlp_local_sgd_cw(int64_t net_kind, Tensor theta_in, std::vector<Tensor> theta_outs, std::vector<Tensor> xs, std::vector<Tensor> ys,
                        std::vector<c10::optional<Tensor>> perms, int64_t batch_size, int64_t epochs, int64_t max_steps, int64_t loss,
                        double lr, int64_t variant, std::vector<double> out_scales, std::vector<double> class_weights) {
  return mlp_fit(net_kind, theta_in, theta_outs, xs, ys, perms, batch_size, epochs, max_steps, loss, lr, variant, out_scales, false,
                 c10::nullopt, 0, 0, c10::nullopt, &class_weights);
}
// the local optimizer instances of mlp_persistent_opt.cu; local_opt: {kind, nesterov, momentum, weight_decay, beta1, beta2, eps}
Tensor mlp_local_sgd_opt(int64_t net_kind, Tensor theta_in, std::vector<Tensor> theta_outs, std::vector<Tensor> xs, std::vector<Tensor> ys,
                         std::vector<c10::optional<Tensor>> perms, int64_t batch_size, int64_t epochs, int64_t max_steps, int64_t loss,
                         double lr, std::vector<double> out_scales, bool delta_mode, c10::optional<Tensor> flags, int64_t perm_seed,
                         int64_t perm_row0, std::vector<double> local_opt) {
  return mlp_fit(net_kind, theta_in, theta_outs, xs, ys, perms, batch_size, epochs, max_steps, loss, lr, 1, out_scales, delta_mode,
                 flags, perm_seed, perm_row0, c10::nullopt, nullptr, &local_opt);
}

// local_opt.cuh's per-element step over arrays, in place: g [steps, n] holds the gradient of every step, m and v the moments
void local_opt_steps(Tensor theta, Tensor g, Tensor m, Tensor v, double lr, std::vector<double> o) {
  TORCH_CHECK(o.size() == 7, "local optimizer: 7 values");
  const int64_t n = theta.numel();
  TORCH_CHECK(g.dim() == 2 && g.size(1) == n && m.numel() == n && v.numel() == n, "theta, m, v [n], g [steps, n]");
  const int64_t steps = g.size(0);
  float* t = const_cast<float*>(fptr(theta, "theta"));
  const float* gp = fptr(g, "g");
  float* mp = const_cast<float*>(fptr(m, "m"));
  float* vp = const_cast<float*>(fptr(v, "v"));
  const colearn::LocalOptArgs lo{(int)o[0], (int)o[1], (float)o[2], (float)o[3], (float)o[4], (float)o[5], (float)o[6]};
  colearn::LocalOptStep st = colearn::local_opt_start();
  for (int64_t s = 0; s < steps; ++s) colearn::local_opt_pass(lo, st, (float)lr, t, gp + s * n, mp, vp, n);
}

Tensor mlp_forward(int64_t net_kind, Tensor theta, Tensor x, int64_t d_out) {
  TORCH_CHECK(x.dim() == 2, "x [n, d_in]");
  Tensor out = torch::zeros({x.size(0), d_out}, torch::kFloat);
  {
    py::gil_scoped_release nogil;
    cudaError_t e = colearn::launch_mlp_forward((int)net_kind, fptr(theta, "theta"), fptr(x, "x"), out.data_ptr<float>(), (int)x.size(0), nullptr);
    TORCH_CHECK(e == cudaSuccess, "launch_mlp_forward (host shim) failed");
  }
  return out;
}

// ---- elementwise.cu ---------------------------------------------------------------------------------------------
#define CK(expr) TORCH_CHECK((expr) == cudaSuccess, "launch failed: " #expr)
float* fmut(Tensor& t, const char* name) { return const_cast<float*>(fptr(t, name)); }

void sgd_step(Tensor p, Tensor g, double lr) { CK(colearn::launch_sgd_step(fmut(p, "p"), fptr(g, "g"), (float)lr, p.numel(), nullptr)); }
// server optimizer (server_opt.cuh): kind 0 = plain server_lr; hyper = [beta1, beta2, tau]; m / v: CPU fp32 moment buffers of n floats
colearn::ServerOptArgs server_opt_args(int64_t kind, double lr, const std::vector<double>& hyper, c10::optional<Tensor>& m,
                                       c10::optional<Tensor>& v, int64_t n) {
  colearn::ServerOptArgs o;
  memset(&o, 0, sizeof(o));
  o.kind = (int)kind;
  o.lr = (float)lr;
  if (kind != colearn::SOPT_SGD) {
    TORCH_CHECK(hyper.size() == 3, "hyper = [beta1, beta2, tau]");
    o.beta1 = (float)hyper[0]; o.beta2 = (float)hyper[1]; o.tau = (float)hyper[2];
    if (m.has_value()) { TORCH_CHECK(m->numel() >= n, "m size"); o.m = fmut(*m, "m"); }
    if (v.has_value()) { TORCH_CHECK(v->numel() >= n, "v size"); o.v = fmut(*v, "v"); }
  }
  TORCH_CHECK(colearn::server_opt_args_ok(o), "server optimizer: unknown kind or a moment buffer missing / misaligned");
  return o;
}
// aggregator (robust_agg.cuh): kind 0 = weighted mean; 1 = median, 2 = trimmed mean with `trim` per end
colearn::AggArgs agg_args(int64_t kind, double trim) {
  colearn::AggArgs g;
  memset(&g, 0, sizeof(g));
  g.kind = (int)kind;
  g.trim = (float)trim;
  TORCH_CHECK(colearn::agg_args_ok(g), "aggregator: unknown kind ", kind, " or trim fraction ", trim, " outside [0, 0.5)");
  return g;
}
// the trailing block of every fused FedAvg apply, as bindings.cpp::fedavg_apply_rows: CPU fp32 moments and agg_weights_out [K],
// the work buffer in CPU memory, and the launcher's grid override of the distance-based kinds
void fedavg_apply_rows(Tensor& theta, const colearn::ClientRows& rows, double server_lr, int64_t opt_kind, const std::vector<double>& opt_hyper,
                       c10::optional<Tensor>& m, c10::optional<Tensor>& v, int64_t agg_kind, double trim, int64_t iters, double eps,
                       double clip, c10::optional<Tensor>& agg_weights_out, int64_t grid) {
  const int64_t n = theta.numel();
  const colearn::ServerOptArgs o = server_opt_args(opt_kind, server_lr, opt_hyper, m, v, n);
  const colearn::AggregatorArgs g{(int)agg_kind, (float)trim, (int)iters, (float)eps, (float)clip};
  colearn::ApplyWork w{nullptr, nullptr, (int)grid};
  if (agg_weights_out.has_value()) {
    TORCH_CHECK(agg_weights_out->numel() == rows.k, "agg_weights_out [K]");
    w.weights_out = fmut(*agg_weights_out, "agg_weights_out");
  }
  Tensor scratch;
  if (const size_t bytes = colearn::fedavg_apply_work_bytes(rows, g, n)) {
    scratch = torch::zeros({(int64_t)(bytes + 7) / 8 + 2}, torch::kDouble);
    w.scratch = scratch.data_ptr();
  }
  float* t = fmut(theta, "theta");
  py::gil_scoped_release nogil;
  CK(colearn::launch_fedavg_apply(t, rows, g, o, n, w, nullptr));
}
colearn::ClientRows client_rows(int format, int64_t k, int64_t stride, const float* weights) {
  colearn::ClientRows r{};
  r.format = format;
  r.k = (int)k;
  r.stride = stride;
  r.weights = weights;
  return r;
}
void fedavg_apply(Tensor theta, Tensor slots, Tensor w, double server_lr, int64_t opt_kind, std::vector<double> opt_hyper,
                  c10::optional<Tensor> m, c10::optional<Tensor> v, int64_t agg_kind, double trim, int64_t iters, double eps, double clip,
                  c10::optional<Tensor> agg_weights_out, int64_t grid) {
  // (the rows may be a strided view: slot stride = slots.stride(0))
  TORCH_CHECK(!slots.is_cuda() && slots.scalar_type() == at::kFloat && slots.dim() == 2 && slots.stride(1) == 1 && slots.size(1) >= theta.numel() &&
              w.numel() == slots.size(0), "slots [K, >= P] (unit inner stride), weights [K]");
  colearn::ClientRows r = client_rows(colearn::ROWS_F32, slots.size(0), slots.stride(0), fptr(w, "w"));
  r.models = slots.data_ptr<float>();
  fedavg_apply_rows(theta, r, server_lr, opt_kind, opt_hyper, m, v, agg_kind, trim, iters, eps, clip, agg_weights_out, grid);
}
// asynchronous buffered aggregation: same shapes as bindings.cpp::fedavg_apply_based (base_slot is read by the launcher and the
// kernels alike)
void fedavg_apply_based(Tensor theta, Tensor models, Tensor ring, Tensor base_slot, Tensor w, int64_t write_slot, double server_lr,
                        int64_t opt_kind, std::vector<double> opt_hyper, c10::optional<Tensor> m, c10::optional<Tensor> v, int64_t agg_kind,
                        double trim, int64_t iters, double eps, double clip, c10::optional<Tensor> agg_weights_out, int64_t grid) {
  TORCH_CHECK(!models.is_cuda() && models.scalar_type() == at::kFloat && models.dim() == 2 && models.stride(1) == 1 &&
              models.size(1) >= theta.numel() && w.numel() == models.size(0), "models [K, >= P] (unit inner stride), weights [K]");
  TORCH_CHECK(ring.dim() == 2 && ring.size(1) == theta.numel() && ring.is_contiguous(), "ring: contiguous [slots, P]");
  TORCH_CHECK(base_slot.scalar_type() == at::kInt && base_slot.is_contiguous() && base_slot.numel() == models.size(0), "base_slot int32 [K]");
  colearn::ClientRows r = client_rows(colearn::ROWS_F32_BASED, models.size(0), models.stride(0), fptr(w, "w"));
  r.models = models.data_ptr<float>();
  r.ring = fmut(ring, "ring");
  r.ring_slots = (int)ring.size(0);
  r.write_slot = (int)write_slot;
  r.base_slot = r.base_slot_host = base_slot.data_ptr<int>();
  fedavg_apply_rows(theta, r, server_lr, opt_kind, opt_hyper, m, v, agg_kind, trim, iters, eps, clip, agg_weights_out, grid);
}
// uplink codec (uplink_quant.cuh): same shapes and row padding as bindings.cpp::quantize_delta / fedavg_apply_quantized
std::tuple<Tensor, Tensor> quantize_delta(Tensor models, Tensor theta, Tensor keys, int64_t bits) {
  TORCH_CHECK(models.dim() == 2 && models.size(1) == theta.numel(), "models [K, P], theta [P]");
  TORCH_CHECK(!keys.is_cuda() && keys.scalar_type() == at::kInt && keys.is_contiguous() && keys.numel() == models.size(0), "keys int32 [K]");
  const int64_t k = models.size(0), n = theta.numel();
  const int64_t row = ((bits == 8 ? n : (n + 1) / 2) + 15) / 16 * 16;
  Tensor payload = torch::zeros({k, row}, torch::kUInt8), scales = torch::zeros({k, (n + 255) / 256}, torch::kFloat);
  {
    py::gil_scoped_release nogil;
    CK(colearn::launch_quantize_delta(fptr(models, "models"), models.stride(0), fptr(theta, "theta"),
                                      reinterpret_cast<const uint32_t*>(keys.data_ptr<int>()), (int)k, (int)bits, payload.data_ptr<uint8_t>(), row,
                                      scales.data_ptr<float>(), n, nullptr));
  }
  return {payload, scales};
}
void fedavg_apply_quantized(Tensor theta, Tensor payload, Tensor scales, Tensor w, int64_t bits, double server_lr, int64_t opt_kind,
                            std::vector<double> opt_hyper, c10::optional<Tensor> m, c10::optional<Tensor> v, int64_t agg_kind, double trim,
                            int64_t iters, double eps, double clip, c10::optional<Tensor> agg_weights_out, int64_t grid) {
  TORCH_CHECK(!payload.is_cuda() && payload.scalar_type() == at::kByte && payload.dim() == 2 && payload.stride(1) == 1, "payload uint8 [K, row]");
  const int64_t k = payload.size(0), n = theta.numel();
  TORCH_CHECK(scales.size(0) == k && scales.size(1) == (n + 255) / 256 && w.numel() == k, "scales [K, ceil(P / 256)], weights [K]");
  TORCH_CHECK(bits == 8 || bits == 4, "bits must be 8 or 4");
  colearn::ClientRows r = client_rows(bits == 8 ? colearn::ROWS_INT8 : colearn::ROWS_INT4, k, payload.stride(0), fptr(w, "w"));
  r.payload = payload.data_ptr<uint8_t>();
  r.scales = fptr(scales, "scales");
  fedavg_apply_rows(theta, r, server_lr, opt_kind, opt_hyper, m, v, agg_kind, trim, iters, eps, clip, agg_weights_out, grid);
}
// top-k uplink (uplink_topk.cuh): same shapes as bindings.cpp::topk_delta / fedavg_apply_topk; residual [K, P] updated in place
std::tuple<Tensor, Tensor> topk_delta(Tensor models, Tensor theta, Tensor residual, int64_t topk) {
  TORCH_CHECK(models.dim() == 2 && models.size(1) == theta.numel() && residual.sizes() == models.sizes(), "models / residual [K, P], theta [P]");
  TORCH_CHECK(topk >= 1 && topk <= colearn::kUtMaxK, "topk must be in 1..32");
  const int64_t k = models.size(0), n = theta.numel(), e = colearn::ut_entries(n, (int)topk);
  Tensor indices = torch::zeros({k, e}, torch::kUInt8), values = torch::zeros({k, e}, torch::kFloat);
  float* res = fmut(residual, "residual");
  {
    py::gil_scoped_release nogil;
    CK(colearn::launch_topk_delta(fptr(models, "models"), models.stride(0), fptr(theta, "theta"), res, n, (int)k, (int)topk,
                                  indices.data_ptr<uint8_t>(), values.data_ptr<float>(), e, n, nullptr));
  }
  return {indices, values};
}
void fedavg_apply_topk(Tensor theta, Tensor indices, Tensor values, Tensor w, int64_t topk, double server_lr, int64_t opt_kind,
                       std::vector<double> opt_hyper, c10::optional<Tensor> m, c10::optional<Tensor> v, int64_t agg_kind, double trim,
                       int64_t iters, double eps, double clip, c10::optional<Tensor> agg_weights_out, int64_t grid) {
  TORCH_CHECK(!indices.is_cuda() && indices.scalar_type() == at::kByte && indices.dim() == 2 && indices.is_contiguous(), "indices uint8 [K, E]");
  const int64_t k = indices.size(0), n = theta.numel();
  TORCH_CHECK(topk >= 1 && topk <= colearn::kUtMaxK && indices.size(1) == colearn::ut_entries(n, (int)topk) &&
              values.sizes() == indices.sizes() && w.numel() == k, "indices / values [K, E(P, topk)], weights [K]");
  colearn::ClientRows r = client_rows(colearn::ROWS_TOPK, k, indices.size(1), fptr(w, "w"));
  r.indices = indices.data_ptr<uint8_t>();
  r.values = fptr(values, "values");
  r.topk = (int)topk;
  fedavg_apply_rows(theta, r, server_lr, opt_kind, opt_hyper, m, v, agg_kind, trim, iters, eps, clip, agg_weights_out, grid);
}
// compressed downlink (downlink.cuh): same shapes and padding as bindings.cpp::downlink_quant / downlink_topk /
// replica_apply_quant / replica_apply_topk; the replica [P] is advanced in place
std::tuple<Tensor, Tensor> downlink_quant(Tensor theta, Tensor replica, int64_t key, int64_t bits) {
  TORCH_CHECK(replica.numel() == theta.numel(), "theta / replica [P]");
  const int64_t n = theta.numel();
  const int64_t row = ((bits == 8 ? n : (n + 1) / 2) + 15) / 16 * 16;
  Tensor payload = torch::zeros({row}, torch::kUInt8), scales = torch::zeros({(n + 255) / 256}, torch::kFloat);
  float* r = fmut(replica, "replica");
  {
    py::gil_scoped_release nogil;
    CK(colearn::launch_downlink_quant(fptr(theta, "theta"), r, (uint32_t)key, (int)bits, payload.data_ptr<uint8_t>(), row,
                                      scales.data_ptr<float>(), n, nullptr));
  }
  return {payload, scales};
}
std::tuple<Tensor, Tensor> downlink_topk(Tensor theta, Tensor replica, int64_t topk) {
  TORCH_CHECK(replica.numel() == theta.numel(), "theta / replica [P]");
  TORCH_CHECK(topk >= 1 && topk <= colearn::kUtMaxK, "topk must be in 1..32");
  const int64_t n = theta.numel(), e = colearn::ut_entries(n, (int)topk);
  Tensor indices = torch::zeros({e}, torch::kUInt8), values = torch::zeros({e}, torch::kFloat);
  float* r = fmut(replica, "replica");
  {
    py::gil_scoped_release nogil;
    CK(colearn::launch_downlink_topk(fptr(theta, "theta"), r, (int)topk, indices.data_ptr<uint8_t>(), values.data_ptr<float>(), n, nullptr));
  }
  return {indices, values};
}
void replica_apply_quant(Tensor replica, Tensor payload, Tensor scales, int64_t bits) {
  TORCH_CHECK(!payload.is_cuda() && payload.scalar_type() == at::kByte && payload.dim() == 1 && payload.is_contiguous(), "payload uint8 [row]");
  const int64_t n = replica.numel();
  TORCH_CHECK(scales.numel() == (n + 255) / 256, "scales [ceil(P / 256)]");
  float* r = fmut(replica, "replica");
  py::gil_scoped_release nogil;
  CK(colearn::launch_replica_apply_quant(r, payload.data_ptr<uint8_t>(), payload.numel(), fptr(scales, "scales"), (int)bits, n, nullptr));
}
void replica_apply_topk(Tensor replica, Tensor indices, Tensor values, int64_t topk) {
  TORCH_CHECK(!indices.is_cuda() && indices.scalar_type() == at::kByte && indices.is_contiguous(), "indices uint8 [E]");
  const int64_t n = replica.numel();
  TORCH_CHECK(topk >= 1 && topk <= colearn::kUtMaxK && indices.numel() == colearn::ut_entries(n, (int)topk) &&
              values.numel() == indices.numel(), "indices / values [E(P, topk)]");
  float* r = fmut(replica, "replica");
  py::gil_scoped_release nogil;
  CK(colearn::launch_replica_apply_topk(r, indices.data_ptr<uint8_t>(), fptr(values, "values"), (int)topk, n, nullptr));
}
// secure aggregation (secagg.cuh): same shapes as bindings.cpp::secagg_mask / fedavg_apply_secagg (uint32 words in int32 tensors)
std::tuple<Tensor, Tensor> secagg_mask(Tensor model, Tensor theta, Tensor keys, Tensor signs, double clip, int64_t frac_bits) {
  TORCH_CHECK(model.numel() == theta.numel(), "model / theta [P]");
  TORCH_CHECK(keys.scalar_type() == at::kInt && keys.is_contiguous() && keys.dim() == 2 && keys.size(1) == 8, "keys int32 [S, 8]");
  TORCH_CHECK(signs.scalar_type() == at::kInt && signs.is_contiguous() && signs.numel() == keys.size(0), "signs int32 [S]");
  const int64_t n = theta.numel();
  Tensor out = torch::zeros({n}, torch::kInt), counts = torch::zeros({2}, torch::kInt);
  {
    py::gil_scoped_release nogil;
    CK(colearn::launch_secagg_mask(fptr(model, "model"), fptr(theta, "theta"), reinterpret_cast<const uint32_t*>(keys.data_ptr<int>()),
                                   signs.data_ptr<int>(), (int)keys.size(0), (float)clip, (int)frac_bits,
                                   reinterpret_cast<uint32_t*>(out.data_ptr<int>()), counts.data_ptr<int>(), n, nullptr));
  }
  return {out, counts};
}
void fedavg_apply_secagg(Tensor theta, Tensor masked, Tensor keys, Tensor signs, int64_t frac_bits, int64_t n_mean, double server_lr,
                         int64_t opt_kind, std::vector<double> opt_hyper, c10::optional<Tensor> m, c10::optional<Tensor> v, int64_t agg_kind,
                         double trim, int64_t iters, double eps, double clip, c10::optional<Tensor> agg_weights_out, int64_t grid) {
  TORCH_CHECK(masked.scalar_type() == at::kInt && masked.dim() == 2 && masked.stride(1) == 1 && masked.size(1) >= theta.numel(), "masked int32 [K, >= P]");
  TORCH_CHECK(keys.scalar_type() == at::kInt && keys.is_contiguous() && keys.dim() == 2 && keys.size(1) == 8, "keys int32 [S, 8]");
  TORCH_CHECK(signs.scalar_type() == at::kInt && signs.is_contiguous() && signs.numel() == keys.size(0), "signs int32 [S]");
  colearn::ClientRows r = client_rows(colearn::ROWS_SECAGG, masked.size(0), masked.stride(0), nullptr);
  r.masked = reinterpret_cast<const uint32_t*>(masked.data_ptr<int>());
  r.keys = reinterpret_cast<const uint32_t*>(keys.data_ptr<int>());
  r.signs = signs.data_ptr<int>();
  r.streams = (int)keys.size(0);
  r.frac_bits = (int)frac_bits;
  r.n_mean = (int)n_mean;
  fedavg_apply_rows(theta, r, server_lr, opt_kind, opt_hyper, m, v, agg_kind, trim, iters, eps, clip, agg_weights_out, grid);
}
Tensor fedavg_flat(Tensor slots, Tensor w) {
  Tensor out = torch::zeros({slots.size(1)}, torch::kFloat);
  CK(colearn::launch_fedavg_flat(out.data_ptr<float>(), fptr(slots, "slots"), slots.size(1), fptr(w, "w"), (int)slots.size(0), slots.size(1), nullptr));
  return out;
}
std::tuple<Tensor, Tensor> sigmoid_bce(Tensor z, Tensor y) {
  Tensor dz = torch::zeros_like(z), loss = torch::zeros({}, torch::kFloat);
  CK(colearn::launch_sigmoid_bce(fptr(z, "z"), fptr(y, "y"), dz.data_ptr<float>(), loss.data_ptr<float>(), z.numel(), nullptr));
  return {loss, dz};
}
std::tuple<Tensor, Tensor> sse_loss(Tensor out, Tensor y, double scale) {
  Tensor dz = torch::zeros_like(out), loss = torch::zeros({}, torch::kFloat);
  CK(colearn::launch_sse(fptr(out, "out"), fptr(y, "y"), dz.data_ptr<float>(), loss.data_ptr<float>(), out.numel(), (float)scale, nullptr));
  return {loss, dz};
}
std::tuple<Tensor, Tensor> softmax_xent(Tensor logits, Tensor labels) {
  TORCH_CHECK(logits.dim() == 2 && labels.scalar_type() == at::kLong && labels.numel() == logits.size(0), "logits [R, C], labels int64 [R]");
  Tensor dl = torch::zeros_like(logits), loss = torch::zeros({}, torch::kFloat);
  CK(colearn::launch_softmax_xent(fptr(logits, "logits"), 0, labels.data_ptr<int64_t>(), dl.data_ptr<float>(), nullptr, loss.data_ptr<float>(),
                                  (int)logits.size(0), (int)logits.size(1), nullptr));
  return {loss, dl};
}
Tensor softmax_xent_head(Tensor logits, Tensor labels, int64_t rows, int64_t cols, c10::optional<Tensor> dl_f32, c10::optional<Tensor> dl_bf16,
                         c10::optional<Tensor> db) {
  TORCH_CHECK(!logits.is_cuda() && logits.dim() == 2 && logits.stride(1) == 1 && labels.scalar_type() == at::kLong && labels.is_contiguous(), "operands");
  const bool bf16 = logits.scalar_type() == at::kBFloat16;
  Tensor loss = torch::zeros({}, torch::kFloat);
  CK(colearn::launch_softmax_xent_head(logits.data_ptr(), bf16 ? 1 : 0, (int)logits.stride(0), labels.data_ptr<int64_t>(),
                                       dl_f32.has_value() ? dl_f32->data_ptr<float>() : nullptr, dl_f32.has_value() ? (int)dl_f32->stride(0) : 0,
                                       dl_bf16.has_value() ? dl_bf16->data_ptr() : nullptr, dl_bf16.has_value() ? (int)dl_bf16->stride(0) : 0,
                                       db.has_value() ? db->data_ptr<float>() : nullptr, loss.data_ptr<float>(), (int)rows, (int)cols, nullptr));
  return loss;
}
std::tuple<Tensor, Tensor> eval_binary(Tensor p, Tensor y) {
  Tensor loss = torch::zeros({}, torch::kFloat), correct = torch::zeros({}, torch::kInt);
  CK(colearn::launch_eval_binary(fptr(p, "p"), fptr(y, "y"), loss.data_ptr<float>(), correct.data_ptr<int>(), p.numel(), nullptr));
  return {loss, correct};
}
// detection-metrics summary: same arguments and results as bindings.cpp::eval_summary on CPU tensors; grid <= 0 picks it
std::tuple<Tensor, Tensor> eval_summary(Tensor scores, Tensor labels, Tensor offsets, int64_t bins, double threshold, int64_t grid) {
  TORCH_CHECK(scores.dim() == 2 && labels.dim() == 1 && labels.size(0) == scores.size(0), "scores [N, C], labels [N]");
  TORCH_CHECK(offsets.scalar_type() == at::kLong && offsets.is_contiguous() && offsets.dim() == 1 && offsets.numel() >= 2, "offsets int64 [S + 1]");
  const int C = (int)scores.size(1), S = (int)offsets.numel() - 1;
  TORCH_CHECK(colearn::eval_summary_args_ok(C, (int)bins, (float)threshold), "eval_summary: arguments outside the limits");
  std::vector<int64_t> table;
  const int64_t units = colearn::es_build_table(offsets.data_ptr<int64_t>(), S, table);
  TORCH_CHECK(units >= 0 && table[S] == scores.size(0), "offsets must rise from 0 to N");
  TORCH_CHECK(scores.size(0) <= colearn::kEsMaxRows, "eval_summary: at most 2^32 - 1 rows per launch (uint32 shared-memory counters)");
  Tensor out = torch::empty({colearn::es_out_words(S, C, (int)bins, units)}, torch::kLong);
  colearn::EvalSummaryArgs a{fptr(scores, "scores"), fptr(labels, "labels"), table.data(), S, units, C, (int)bins, (float)threshold,
                             out.data_ptr<int64_t>()};
  {
    py::gil_scoped_release nogil;
    CK(colearn::launch_eval_summary(a, (int)grid, nullptr));
  }
  const int64_t L = colearn::es_row_len(C, (int)bins);
  return {out.narrow(0, 0, S * L).view({S, L}), out.narrow(0, S * L, S).view(at::kDouble)};
}
// reconstruction-error summary: same arguments and results as bindings.cpp::recon_summary on CPU tensors; grid <= 0 picks it
std::vector<Tensor> recon_summary(Tensor xhat, Tensor x, c10::optional<Tensor> labels, Tensor offsets, int64_t bins, int64_t alarm_bin,
                                  int64_t grid) {
  TORCH_CHECK(xhat.dim() == 2 && x.sizes() == xhat.sizes(), "xhat and x: [N, D]");
  TORCH_CHECK(!labels.has_value() || (labels->dim() == 1 && labels->size(0) == x.size(0)), "labels [N]");
  TORCH_CHECK(offsets.scalar_type() == at::kLong && offsets.is_contiguous() && offsets.dim() == 1 && offsets.numel() >= 2, "offsets int64 [S + 1]");
  TORCH_CHECK(x.size(1) <= colearn::kRsMaxDim && colearn::recon_summary_args_ok((int)x.size(1), (int)bins) && bins <= colearn::kRsMaxBins,
              "recon_summary: arguments outside the limits");
  TORCH_CHECK(alarm_bin < 0 || alarm_bin <= bins, "recon_summary: the alarm bin must be in [0, bins]");
  const int S = (int)offsets.numel() - 1;
  std::vector<int64_t> table;
  const int64_t units = colearn::es_build_table(offsets.data_ptr<int64_t>(), S, table);
  TORCH_CHECK(units >= 0 && table[S] == x.size(0), "offsets must rise from 0 to N");
  TORCH_CHECK(x.size(0) <= colearn::kEsMaxRows, "recon_summary: at most 2^32 - 1 rows per launch (uint32 shared-memory counters)");
  Tensor out = torch::empty({colearn::rs_out_words(S, (int)bins, units)}, torch::kLong);
  const bool rows = alarm_bin >= 0;
  Tensor err = torch::empty({rows ? x.size(0) : 0}, torch::kFloat), flag = torch::empty({rows ? x.size(0) : 0}, torch::kUInt8);
  colearn::ReconSummaryArgs a{fptr(xhat, "xhat"), fptr(x, "x"), labels.has_value() ? fptr(*labels, "labels") : nullptr, table.data(), S, units,
                              (int)x.size(1), (int)bins, rows ? (int)alarm_bin : 0, rows ? err.data_ptr<float>() : nullptr,
                              rows ? flag.data_ptr<uint8_t>() : nullptr, out.data_ptr<int64_t>()};
  {
    py::gil_scoped_release nogil;
    CK(colearn::launch_recon_summary(a, (int)grid, nullptr));
  }
  const int64_t L = colearn::rs_row_len((int)bins);
  return {out.narrow(0, 0, S * L).view({S, L}), out.narrow(0, S * L, S).view(at::kDouble), err, flag};
}
Tensor argmax_rows(Tensor x) {
  Tensor out = torch::zeros({x.size(0), 1}, torch::kLong);
  CK(colearn::launch_argmax_rows(fptr(x, "x"), out.data_ptr<int64_t>(), (int)x.size(0), (int)x.size(1), nullptr));
  return out;
}
Tensor minmax_scale(Tensor x) {
  Tensor out = torch::zeros_like(x);
  CK(colearn::launch_minmax_scale(fptr(x, "x"), out.data_ptr<float>(), (int)x.size(0), (int)x.size(1), nullptr));
  return out;
}
Tensor feistel_permutation(int64_t n, int64_t rows, int64_t seed) {
  Tensor out = torch::zeros({rows, n}, torch::kInt);
  CK(colearn::launch_feistel_permutation(out.data_ptr<int>(), (int)n, (int)rows, (uint64_t)seed, nullptr));
  return out;
}
Tensor transpose_bf16(Tensor x) {
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && x.is_contiguous() && x.dim() == 2, "bf16 matrix");
  Tensor out = torch::zeros({x.size(1), x.size(0)}, x.options());
  CK(colearn::launch_transpose_bf16(x.data_ptr(), out.data_ptr(), (int)x.size(0), (int)x.size(1), nullptr));
  return out;
}
Tensor ring_matmul(Tensor a, Tensor b) {
  TORCH_CHECK(a.scalar_type() == at::kLong && b.scalar_type() == at::kLong && a.is_contiguous() && b.is_contiguous(), "int64 matrices");
  Tensor c = torch::zeros({a.size(0), b.size(1)}, torch::kLong);
  CK(colearn::launch_ring_matmul(reinterpret_cast<const long long*>(a.data_ptr<int64_t>()), reinterpret_cast<const long long*>(b.data_ptr<int64_t>()),
                                 reinterpret_cast<long long*>(c.data_ptr<int64_t>()), (int)a.size(0), (int)a.size(1), (int)b.size(1), nullptr));
  return c;
}

// ---- comm.cu: W emulated ranks = W sets of buffers in this process; kernels of different ranks run one after the other -----
// Coordinator-side star round: slots [W, P] (already holding w_k * theta_k), arrive flags int32 [W], inboxes [W, P] (row k =
// rank k's inbox), bcast flags int32 [W].  Returns the arrived mask (deadline mode) or the select mask.
int64_t star_round(Tensor theta, Tensor slots, Tensor arrive, int64_t arrive_epoch, Tensor inboxes, Tensor bcast_flags, int64_t bcast_epoch,
                   int64_t select_mask, double server_lr, bool do_reduce, bool do_bcast, int64_t n_blocks, double timeout_ms,
                   std::vector<double> weights, int64_t opt_kind, std::vector<double> opt_hyper, c10::optional<Tensor> m,
                   c10::optional<Tensor> v, int64_t agg_kind, double trim) {
  const int W = (int)slots.size(0);
  colearn::StarRoundArgs a;
  memset(&a, 0, sizeof(a));
  a.theta = fmut(theta, "theta");
  a.slots = fptr(slots, "slots");
  a.slot_stride = slots.size(1);
  a.arrive_flags = reinterpret_cast<const uint32_t*>(arrive.data_ptr<int>());
  a.arrive_epoch = (uint32_t)arrive_epoch;
  for (int k = 0; k < W; ++k) {
    a.peer_inbox[k] = inboxes.data_ptr<float>() + (int64_t)k * inboxes.size(1);
    a.peer_bcast_flag[k] = reinterpret_cast<uint32_t*>(bcast_flags.data_ptr<int>()) + k;
    a.weights[k] = k < (int)weights.size() ? (float)weights[k] : 0.f;
  }
  a.bcast_epoch = (uint32_t)bcast_epoch;
  a.select_mask = (uint32_t)select_mask;
  a.world = W;
  a.server_lr = (float)server_lr;
  a.n = theta.numel();
  a.do_reduce = do_reduce ? 1 : 0;
  a.do_bcast = do_bcast ? 1 : 0;
  static uint32_t counter = 0, decision[2] = {0, 0};
  a.grid_counter = &counter;
  a.timeout_ns = (unsigned long long)(timeout_ms * 1e6);
  a.decision = decision;
  a.opt = server_opt_args(opt_kind, server_lr, opt_hyper, m, v, a.n);
  a.agg = agg_args(agg_kind, trim);
  {
    py::gil_scoped_release nogil;
    CK(colearn::launch_star_round(a, (int)n_blocks, nullptr));
  }
  return timeout_ms > 0 && do_reduce ? (int64_t)decision[1] : select_mask;
}

// One rank's two-shot kernel (P2P path): works [W, n] (row k = rank k's fp32 arena), shadows [W, n] bf16 or none, chunk flags
// int32 [W, n_chunks]; `arrive` (this rank's int32 [W]) must already carry `epoch` for every selected rank.
void twoshot_fedavg(int64_t rank, Tensor works, c10::optional<Tensor> shadows, Tensor chunk_flags, Tensor arrive, Tensor weights,
                    c10::optional<Tensor> theta_prev, int64_t epoch, int64_t select_mask, double server_lr, int64_t chunk_elems, int64_t n_blocks,
                    c10::optional<Tensor> produced, double produced_timeout_s, int64_t opt_kind, std::vector<double> opt_hyper,
                    c10::optional<Tensor> m, c10::optional<Tensor> v, int64_t agg_kind, double trim) {
  const int W = (int)works.size(0);
  colearn::TwoShotArgs a;
  memset(&a, 0, sizeof(a));
  for (int k = 0; k < W; ++k) {
    a.work[k] = works.data_ptr<float>() + (int64_t)k * works.size(1);
    a.shadow_bf16[k] = shadows.has_value() ? static_cast<void*>(static_cast<char*>(shadows->data_ptr()) + (int64_t)k * shadows->size(1) * 2) : nullptr;
    a.chunk_flags[k] = reinterpret_cast<uint32_t*>(chunk_flags.data_ptr<int>()) + (int64_t)k * chunk_flags.size(1);
  }
  a.arrive_flags = reinterpret_cast<const uint32_t*>(arrive.data_ptr<int>());
  a.weights = fptr(weights, "weights");
  a.theta_prev = theta_prev.has_value() ? theta_prev->data_ptr<float>() : nullptr;
  a.epoch = (uint32_t)epoch;
  a.select_mask = (uint32_t)select_mask;
  a.server_lr = (float)server_lr;
  a.n = works.size(1);
  a.chunk_elems = chunk_elems;
  a.world = W;
  a.rank = (int)rank;
  if (produced.has_value()) {      // [W (owner), W (producer), n_chunks] int32: this rank's table is produced[rank]
    TORCH_CHECK(produced->dim() == 3 && produced->size(0) == W && produced->size(1) == W && produced->is_contiguous(), "produced");
    a.produced = reinterpret_cast<const uint32_t*>(produced->data_ptr<int>()) + rank * W * produced->size(2);
    a.produced_timeout_ns = produced_timeout_s > 0 ? (unsigned long long)(produced_timeout_s * 1e9) : 0ull;
  }
  a.opt = server_opt_args(opt_kind, server_lr, opt_hyper, m, v, a.n);     // this rank's moment buffers (it touches the chunks it owns)
  TORCH_CHECK(a.opt.kind == colearn::SOPT_SGD || a.theta_prev != nullptr, "a server optimizer needs theta_prev");
  a.agg = agg_args(agg_kind, trim);
  {
    py::gil_scoped_release nogil;
    CK(colearn::launch_twoshot_fedavg(a, (int)n_blocks, nullptr));
  }
}

// deadline mode of one emulated rank: decisions int32 [W, 16] (row k = rank k's ring), globals [W, n] (second arenas)
void twoshot_fedavg_deadline(int64_t rank, Tensor works, Tensor globals, Tensor chunk_flags, Tensor arrive, Tensor weights, int64_t epoch,
                             int64_t select_mask, int64_t chunk_elems, int64_t n_blocks, double deadline_ms, Tensor decisions,
                             int64_t agg_kind, double trim) {
  const int W = (int)works.size(0);
  colearn::TwoShotArgs a;
  memset(&a, 0, sizeof(a));
  for (int k = 0; k < W; ++k) {
    a.work[k] = works.data_ptr<float>() + (int64_t)k * works.size(1);
    a.global_copy[k] = globals.data_ptr<float>() + (int64_t)k * globals.size(1);
    a.chunk_flags[k] = reinterpret_cast<uint32_t*>(chunk_flags.data_ptr<int>()) + (int64_t)k * chunk_flags.size(1);
    a.decision[k] = reinterpret_cast<uint32_t*>(decisions.data_ptr<int>()) + (int64_t)k * decisions.size(1);
  }
  a.arrive_flags = reinterpret_cast<const uint32_t*>(arrive.data_ptr<int>());
  a.weights = a.true_weights = fptr(weights, "weights");
  a.epoch = (uint32_t)epoch;
  a.select_mask = (uint32_t)select_mask;
  a.server_lr = 1.f;
  a.n = works.size(1);
  a.chunk_elems = chunk_elems;
  a.world = W;
  a.rank = (int)rank;
  a.wait_all = 0;      // (the emulated ranks run one after the other: nobody may wait for a later rank's chunks)
  a.deadline_ns = (unsigned long long)(deadline_ms * 1e6);
  a.agg = agg_args(agg_kind, trim);
  py::gil_scoped_release nogil;
  CK(colearn::launch_twoshot_fedavg(a, (int)n_blocks, nullptr));
}

void twoshot_resync(Tensor decision_ring, int64_t prev_epoch, int64_t rank, Tensor work, Tensor global_copy) {
  py::gil_scoped_release nogil;
  CK(colearn::launch_twoshot_resync(reinterpret_cast<const uint32_t*>(decision_ring.data_ptr<int>()), (uint32_t)prev_epoch, (int)rank,
                                    work.data_ptr<float>(), nullptr, global_copy.data_ptr<float>(), work.numel(), 2, nullptr));
}

void reduce_push(Tensor slots, Tensor dst, Tensor losses, Tensor loss_dst, Tensor flag, int64_t value, int64_t n_blocks) {
  static uint32_t counter = 0;
  py::gil_scoped_release nogil;
  CK(colearn::launch_reduce_push(fptr(slots, "slots"), (int)slots.size(0), slots.size(1), slots.size(1), fmut(dst, "dst"), fptr(losses, "losses"),
                                 fmut(loss_dst, "loss_dst"), reinterpret_cast<uint32_t*>(flag.data_ptr<int>()), (uint32_t)value, &counter,
                                 (int)n_blocks, nullptr));
}

#include "produced_bindings.inc"
void produced_mark(int64_t sig, int64_t chunk_elems, int64_t lo, int64_t hi) {
  int shift = 0;
  while (((int64_t)1 << shift) < chunk_elems) ++shift;
  py::gil_scoped_release nogil;
  CK(colearn::launch_produced_mark(reinterpret_cast<const colearn::ProducedSignal*>(static_cast<uintptr_t>(sig)), shift, lo, hi, nullptr));
}

// ---- gemm_wgmma.cu on the functional wgmma / TMA / mbarrier model (gemm_host_model.h) -------------------------------------
// Same argument meaning as bindings.cpp::gemm_tcgen05 (minus the cross-GPU ready flags and the cluster modes).
static void gemm_run(Tensor A, Tensor B, c10::optional<Tensor> bias, bool relu, c10::optional<Tensor> relu_mask, c10::optional<Tensor> out_bf16,
                     c10::optional<Tensor> out_f32, c10::optional<Tensor> out_bf16_t, c10::optional<Tensor> sgd_master, double sgd_lr,
                     c10::optional<Tensor> sgd_shadow, c10::optional<Tensor> sgd_shadow_t, c10::optional<Tensor> colsum, int64_t tile_n,
                     int64_t split_k, c10::optional<Tensor> split_out, int64_t mn_m, bool b_kn, c10::optional<Tensor> addend,
                     std::vector<int64_t> conv, std::vector<int64_t> produced, const colearn::GemmOptEpilogue* lopt) {
  TORCH_CHECK(!A.is_cuda() && !B.is_cuda() && A.scalar_type() == at::kBFloat16 && B.scalar_type() == at::kBFloat16 && A.is_contiguous() &&
              B.is_contiguous() && A.dim() == 2 && B.dim() == 2, "A, B: contiguous CPU bf16 matrices");
  const bool mn = mn_m > 0, is_conv = !conv.empty();
  TORCH_CHECK(!is_conv || conv.size() == 14, "conv = 14 ints");
  const int M = is_conv ? (int)conv[10] : (mn ? (int)mn_m : (int)A.size(0));
  const int N = is_conv ? (int)conv[11] : ((mn || b_kn) ? (int)B.size(1) : (int)B.size(0));
  const int K = is_conv ? (int)conv[12] : (mn ? (int)A.size(0) : (int)A.size(1));
  colearn::GemmEpilogue ep;
  memset(&ep, 0, sizeof(ep));
  auto ptr = [&](const c10::optional<Tensor>& t, at::ScalarType st, int64_t numel, const char* name) -> void* {
    if (!t.has_value()) return nullptr;
    TORCH_CHECK(!t->is_cuda() && t->scalar_type() == st && t->is_contiguous() && t->numel() >= numel, name, ": dtype / size");
    return t->data_ptr();
  };
  ep.bias = (const float*)ptr(bias, at::kFloat, N, "bias");
  ep.relu = relu ? 1 : 0;
  ep.relu_mask = ptr(relu_mask, at::kBFloat16, (int64_t)M * N, "relu_mask");
  ep.out_bf16 = ptr(out_bf16, at::kBFloat16, (int64_t)M * N, "out_bf16");
  ep.out_f32 = (float*)ptr(out_f32, at::kFloat, (int64_t)M * N, "out_f32");
  ep.out_bf16_t = ptr(out_bf16_t, at::kBFloat16, (int64_t)M * N, "out_bf16_t");
  ep.sgd_master = (float*)ptr(sgd_master, at::kFloat, (int64_t)M * N, "sgd_master");
  ep.sgd_lr = (float)sgd_lr;
  ep.sgd_shadow = ptr(sgd_shadow, at::kBFloat16, (int64_t)M * N, "sgd_shadow");
  ep.sgd_shadow_t = ptr(sgd_shadow_t, at::kBFloat16, (int64_t)M * N, "sgd_shadow_t");
  ep.colsum = (float*)ptr(colsum, at::kFloat, (int64_t)(M / 32) * N, "colsum");
  ep.addend = ptr(addend, at::kBFloat16, (int64_t)M * N, "addend");
  if (lopt != nullptr) ep.lopt = *lopt;
  ep.ready_chunk_elems = 1;
  ep.tile_n = (int)tile_n;
  if (!produced.empty()) {
    TORCH_CHECK(produced.size() == 3, "produced = [signal_ptr, elem_offset, max_ctas]");
    ep.produced = reinterpret_cast<const colearn::ProducedSignal*>(static_cast<uintptr_t>(produced[0]));
    ep.produced_elem_offset = produced[1];
    ep.max_ctas = (int)produced[2];
  }
  if (split_k > 1) {
    ep.split_k = (int)split_k;
    ep.split_out = (float*)ptr(split_out, at::kFloat, split_k * (int64_t)M * N, "split_out");
    TORCH_CHECK(ep.split_out != nullptr, "split_out");
  }
  cudaError_t e;
  {
    py::gil_scoped_release nogil;
    if (is_conv) {
      colearn::convops::ConvAddr& g = ep.conv;
      g.mode = (int)conv[0]; g.flip = (int)conv[1]; g.C = (int)conv[2]; g.KH = (int)conv[3]; g.KW = (int)conv[4]; g.pad = (int)conv[5];
      const int H = (int)conv[6], W = (int)conv[7];
      g.HW = H * W; g.n_images = (int)conv[8]; g.b_rows_per_tap = (int)conv[9]; g.b_mn = (int)conv[13];
      e = colearn::launch_gemm_tcgen05_conv(A.data_ptr(), g.n_images, H, W, B.data_ptr(), (int)B.size(0), (int)B.size(1), M, N, K, ep, nullptr);
    } else if (mn || b_kn) {
      e = colearn::launch_gemm_tcgen05_mn(A.data_ptr(), mn ? 1 : 0, (int)A.size(1), B.data_ptr(), (int)B.size(0), M, N, K, ep, nullptr);
    } else {
      e = colearn::launch_gemm_tcgen05(A.data_ptr(), B.data_ptr(), M, N, K, ep, nullptr);
    }
  }
  TORCH_CHECK(e == cudaSuccess, "gemm_tcgen05 (host model): ", colearn::gemm_tcgen05_last_error());
}
void gemm_tcgen05(Tensor A, Tensor B, c10::optional<Tensor> bias, bool relu, c10::optional<Tensor> relu_mask, c10::optional<Tensor> out_bf16,
                  c10::optional<Tensor> out_f32, c10::optional<Tensor> out_bf16_t, c10::optional<Tensor> sgd_master, double sgd_lr,
                  c10::optional<Tensor> sgd_shadow, c10::optional<Tensor> sgd_shadow_t, c10::optional<Tensor> colsum, int64_t tile_n,
                  int64_t split_k, c10::optional<Tensor> split_out, int64_t mn_m, bool b_kn, c10::optional<Tensor> addend,
                  std::vector<int64_t> conv, std::vector<int64_t> produced) {
  gemm_run(A, B, bias, relu, relu_mask, out_bf16, out_f32, out_bf16_t, sgd_master, sgd_lr, sgd_shadow, sgd_shadow_t, colsum, tile_n, split_k,
           split_out, mn_m, b_kn, addend, conv, produced, nullptr);
}

// the local optimizer of the layer-wise trainer (bindings.cpp): opt = {kind, nesterov, momentum, weight_decay, beta1, beta2, eps},
// step = {t, p1, p2, s, r}; m / v: fp32 with the parameter's sizes and strides, None where the optimizer keeps none
static colearn::LocalOptArgs local_opt_args(const std::vector<double>& o) {
  TORCH_CHECK(o.size() == 7, "local optimizer: 7 values");
  TORCH_CHECK((int)o[0] == colearn::LOCAL_OPT_SGD || (int)o[0] == colearn::LOCAL_OPT_ADAM, "local optimizer: unknown kind");
  return colearn::LocalOptArgs{(int)o[0], (int)o[1], (float)o[2], (float)o[3], (float)o[4], (float)o[5], (float)o[6]};
}
static colearn::LocalOptStep local_opt_step_of(const std::vector<double>& step) {
  TORCH_CHECK(step.size() == 5 && step[0] >= 1, "local optimizer step: {t >= 1, p1, p2, s, r}");
  colearn::LocalOptStep st;
  st.t = (int)step[0]; st.p1 = (float)step[1]; st.p2 = (float)step[2]; st.s = (float)step[3]; st.r = (float)step[4];
  return st;
}
static float* local_opt_moment(const c10::optional<Tensor>& t, const Tensor& param, bool needed, const char* name) {
  TORCH_CHECK(t.has_value() || !needed, name, ": this optimizer keeps it, pass the buffer");
  if (!t.has_value()) return nullptr;
  TORCH_CHECK(!t->is_cuda() && t->scalar_type() == at::kFloat && t->sizes() == param.sizes() && t->strides() == param.strides(),
              name, ": CPU fp32 with the parameter's sizes and strides");
  return t->data_ptr<float>();
}
void gemm_tcgen05_opt(Tensor A, Tensor B, c10::optional<Tensor> bias, bool relu, c10::optional<Tensor> relu_mask, c10::optional<Tensor> out_bf16,
                      c10::optional<Tensor> out_f32, c10::optional<Tensor> out_bf16_t, c10::optional<Tensor> sgd_master, double sgd_lr,
                      c10::optional<Tensor> sgd_shadow, c10::optional<Tensor> sgd_shadow_t, c10::optional<Tensor> colsum, int64_t tile_n,
                      int64_t split_k, c10::optional<Tensor> split_out, int64_t mn_m, bool b_kn, c10::optional<Tensor> addend,
                      std::vector<int64_t> conv, std::vector<int64_t> produced, c10::optional<Tensor> m, c10::optional<Tensor> v,
                      std::vector<double> opt, std::vector<double> step) {
  TORCH_CHECK(sgd_master.has_value(), "the local optimizer epilogue updates sgd_master");
  colearn::GemmOptEpilogue lo;
  memset(&lo, 0, sizeof(lo));
  lo.args = local_opt_args(opt);
  lo.step = local_opt_step_of(step);
  lo.m = local_opt_moment(m, *sgd_master, lo.args.kind == colearn::LOCAL_OPT_ADAM || lo.args.momentum != 0.f, "m");
  lo.v = local_opt_moment(v, *sgd_master, lo.args.kind == colearn::LOCAL_OPT_ADAM, "v");
  gemm_run(A, B, bias, relu, relu_mask, out_bf16, out_f32, out_bf16_t, sgd_master, sgd_lr, sgd_shadow, sgd_shadow_t, colsum, tile_n, split_k,
           split_out, mn_m, b_kn, addend, conv, produced, &lo);
}
// local_opt_apply_kernel of elementwise.cu (bindings.cpp::local_opt_apply)
void local_opt_apply(Tensor theta, Tensor grad, int64_t g_rows, c10::optional<Tensor> m, c10::optional<Tensor> v, double lr,
                     std::vector<double> opt, std::vector<double> step) {
  TORCH_CHECK(!theta.is_cuda() && theta.scalar_type() == at::kFloat && theta.dim() == 2 && theta.stride(1) == 1, "theta: CPU fp32 [rows, cols]");
  TORCH_CHECK(!grad.is_cuda() && grad.scalar_type() == at::kFloat && grad.dim() == 2 && grad.stride(1) == 1 && g_rows >= 1 &&
              grad.size(0) == theta.size(0) * g_rows && grad.size(1) >= theta.size(1), "grad: CPU fp32 [rows * g_rows, >= cols]");
  const colearn::LocalOptArgs a = local_opt_args(opt);
  float* mp = local_opt_moment(m, theta, a.kind == colearn::LOCAL_OPT_ADAM || a.momentum != 0.f, "m");
  float* vp = local_opt_moment(v, theta, a.kind == colearn::LOCAL_OPT_ADAM, "v");
  const colearn::LocalOptStep st = local_opt_step_of(step);
  py::gil_scoped_release nogil;
  CK(colearn::launch_local_opt_apply(theta.data_ptr<float>(), theta.stride(0), grad.data_ptr<float>(), grad.stride(0), (int)g_rows, mp, vp,
                                     (int)theta.size(0), (int)theta.size(1), a, st, (float)lr, nullptr));
}

// ---- convnet.cu: the launchers themselves (grid mapping, two-phase blocks, the ticket-counter BatchNorm reduction) behind the
// torch-facing wrappers of conv_bindings.inc — a third instantiation next to the GPU one and the body emulator ----------------
inline void ck(cudaError_t e, const char* what) { TORCH_CHECK(e == cudaSuccess, what, " failed"); }
struct ConvSimtExec {
  static constexpr bool kCuda = false;
  static void im2col(const colearn::convops::Im2colArgs& a) { ck(colearn::launch_im2col(a, nullptr), "im2col"); }
  static void col2im(const colearn::convops::Col2imArgs& a) { ck(colearn::launch_col2im(a, nullptr), "col2im"); }
  static void bn_reduce(const colearn::convops::BnReduceArgs& a) { ck(colearn::launch_bn_reduce(a, nullptr), "bn_reduce"); }
  static void bn_finalize(const colearn::convops::BnFinalizeArgs& a) { ck(colearn::launch_bn_finalize(a, nullptr), "bn_finalize"); }
  static void bn_reduce_finalize(const colearn::convops::BnFusedArgs& a) { ck(colearn::launch_bn_reduce_finalize(a, nullptr), "bn_reduce_finalize"); }
  static void bn_apply(const colearn::convops::BnApplyArgs& a) { ck(colearn::launch_bn_apply(a, nullptr), "bn_apply"); }
  static void bn_bwd(const colearn::convops::BnBwdArgs& a) { ck(colearn::launch_bn_bwd(a, nullptr), "bn_bwd"); }
  static void maxpool_fwd(const colearn::convops::PoolArgs& a) { ck(colearn::launch_maxpool_fwd(a, nullptr), "maxpool_fwd"); }
  static void maxpool_bwd(const colearn::convops::PoolArgs& a) { ck(colearn::launch_maxpool_bwd(a, nullptr), "maxpool_bwd"); }
  static void avgpool_fwd(const colearn::convops::AvgPoolArgs& a) { ck(colearn::launch_avgpool_fwd(a, nullptr), "avgpool_fwd"); }
  static void avgpool_bwd(const colearn::convops::AvgPoolArgs& a) { ck(colearn::launch_avgpool_bwd(a, nullptr), "avgpool_bwd"); }
  static void pack(const colearn::convops::PackArgs& a) { ck(colearn::launch_pack(a, nullptr), "pack"); }
  static void splitk_reduce(const colearn::convops::SplitKReduceArgs& a) { ck(colearn::launch_splitk_reduce(a, nullptr), "splitk_reduce"); }
};
}  // namespace

#include "conv_bindings.inc"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "the CUDA kernels of mlp_persistent.cu / elementwise.cu / comm.cu / convnet.cu compiled for the CPU through a SIMT shim (tests only)";
  convbind::register_ops<ConvSimtExec>(m);
  m.def("gemm_tcgen05", &gemm_tcgen05);
  m.def("gemm_tcgen05_opt", &gemm_tcgen05_opt);
  m.def("local_opt_apply", &local_opt_apply);
  m.def("mlp_local_sgd", &mlp_local_sgd, py::arg("net_kind"), py::arg("theta_in"), py::arg("theta_outs"), py::arg("xs"), py::arg("ys"), py::arg("perms"),
        py::arg("batch_size"), py::arg("epochs"), py::arg("max_steps"), py::arg("loss"), py::arg("lr"), py::arg("variant"), py::arg("out_scales"),
        py::arg("delta_mode"), py::arg("flags"), py::arg("perm_seed") = 0, py::arg("perm_row0") = 0, py::arg("perm_scratch") = py::none());
  m.def("mlp_local_sgd_cw", &mlp_local_sgd_cw);
  m.def("mlp_local_sgd_opt", &mlp_local_sgd_opt);
  m.def("local_opt_steps", &local_opt_steps);
  m.def("mlp_forward", &mlp_forward);
  m.def("mlp_net_params", [](int64_t kind) { return (int64_t)colearn::mlp_net_num_params((int)kind); });
  m.def("sgd_step", &sgd_step);
  // trailing server-optimizer arguments default to plain FedAvg (the shorter positional calls keep working)
  m.def("fedavg_apply", &fedavg_apply, py::arg("theta"), py::arg("slots"), py::arg("w"), py::arg("server_lr"), py::arg("opt_kind") = 0,
        py::arg("opt_hyper") = std::vector<double>{}, py::arg("m") = py::none(), py::arg("v") = py::none(), py::arg("agg_kind") = 0,
        py::arg("trim") = 0.0, py::arg("iters") = 3,
        py::arg("eps") = 1e-6, py::arg("clip") = 0.0, py::arg("agg_weights_out") = py::none(), py::arg("grid") = 0);
  m.def("fedavg_apply_based", &fedavg_apply_based, py::arg("theta"), py::arg("models"), py::arg("ring"), py::arg("base_slot"), py::arg("w"),
        py::arg("write_slot"), py::arg("server_lr"), py::arg("opt_kind") = 0, py::arg("opt_hyper") = std::vector<double>{},
        py::arg("m") = py::none(), py::arg("v") = py::none(), py::arg("agg_kind") = 0, py::arg("trim") = 0.0, py::arg("iters") = 3,
        py::arg("eps") = 1e-6, py::arg("clip") = 0.0, py::arg("agg_weights_out") = py::none(), py::arg("grid") = 0);
  m.def("topk_delta", &topk_delta);
  m.def("fedavg_apply_topk", &fedavg_apply_topk, py::arg("theta"), py::arg("indices"), py::arg("values"), py::arg("w"), py::arg("topk"),
        py::arg("server_lr"), py::arg("opt_kind") = 0, py::arg("opt_hyper") = std::vector<double>{}, py::arg("m") = py::none(),
        py::arg("v") = py::none(), py::arg("agg_kind") = 0, py::arg("trim") = 0.0, py::arg("iters") = 3, py::arg("eps") = 1e-6,
        py::arg("clip") = 0.0, py::arg("agg_weights_out") = py::none(), py::arg("grid") = 0);
  m.def("downlink_quant", &downlink_quant);
  m.def("downlink_topk", &downlink_topk);
  m.def("replica_apply_quant", &replica_apply_quant);
  m.def("replica_apply_topk", &replica_apply_topk);
  m.def("quantize_delta", &quantize_delta);
  m.def("fedavg_apply_quantized", &fedavg_apply_quantized, py::arg("theta"), py::arg("payload"), py::arg("scales"), py::arg("w"),
        py::arg("bits"), py::arg("server_lr"), py::arg("opt_kind") = 0, py::arg("opt_hyper") = std::vector<double>{},
        py::arg("m") = py::none(), py::arg("v") = py::none(), py::arg("agg_kind") = 0, py::arg("trim") = 0.0, py::arg("iters") = 3,
        py::arg("eps") = 1e-6, py::arg("clip") = 0.0, py::arg("agg_weights_out") = py::none(), py::arg("grid") = 0);
  m.def("secagg_mask", &secagg_mask);
  m.def("fedavg_apply_secagg", &fedavg_apply_secagg, py::arg("theta"), py::arg("masked"), py::arg("keys"), py::arg("signs"),
        py::arg("frac_bits"), py::arg("n_mean"), py::arg("server_lr"), py::arg("opt_kind") = 0,
        py::arg("opt_hyper") = std::vector<double>{}, py::arg("m") = py::none(), py::arg("v") = py::none(), py::arg("agg_kind") = 0,
        py::arg("trim") = 0.0, py::arg("iters") = 3, py::arg("eps") = 1e-6, py::arg("clip") = 0.0, py::arg("agg_weights_out") = py::none(),
        py::arg("grid") = 0);
  m.def("fedavg_flat", &fedavg_flat);
  m.def("sigmoid_bce", &sigmoid_bce);
  m.def("sse_loss", &sse_loss);
  m.def("softmax_xent", &softmax_xent);
  m.def("softmax_xent_head", &softmax_xent_head);
  m.def("eval_binary", &eval_binary);
  m.def("eval_summary", &eval_summary);
  m.def("recon_summary", &recon_summary);
  m.def("argmax_rows", &argmax_rows);
  m.def("minmax_scale", &minmax_scale);
  m.def("feistel_permutation", &feistel_permutation);
  m.def("transpose_bf16", &transpose_bf16);
  m.def("ring_matmul", &ring_matmul);
  m.def("star_round", &star_round, py::arg("theta"), py::arg("slots"), py::arg("arrive"), py::arg("arrive_epoch"), py::arg("inboxes"),
        py::arg("bcast_flags"), py::arg("bcast_epoch"), py::arg("select_mask"), py::arg("server_lr"), py::arg("do_reduce"), py::arg("do_bcast"),
        py::arg("n_blocks"), py::arg("timeout_ms"), py::arg("weights"), py::arg("opt_kind") = 0, py::arg("opt_hyper") = std::vector<double>{},
        py::arg("m") = py::none(), py::arg("v") = py::none(), py::arg("agg_kind") = 0, py::arg("trim") = 0.0);
  m.def("twoshot_fedavg", &twoshot_fedavg, py::arg("rank"), py::arg("works"), py::arg("shadows"), py::arg("chunk_flags"), py::arg("arrive"),
        py::arg("weights"), py::arg("theta_prev"), py::arg("epoch"), py::arg("select_mask"), py::arg("server_lr"), py::arg("chunk_elems"),
        py::arg("n_blocks"), py::arg("produced"), py::arg("produced_timeout_s"), py::arg("opt_kind") = 0,
        py::arg("opt_hyper") = std::vector<double>{}, py::arg("m") = py::none(), py::arg("v") = py::none(), py::arg("agg_kind") = 0,
        py::arg("trim") = 0.0);
  m.def("twoshot_fedavg_deadline", &twoshot_fedavg_deadline, py::arg("rank"), py::arg("works"), py::arg("globals"), py::arg("chunk_flags"),
        py::arg("arrive"), py::arg("weights"), py::arg("epoch"), py::arg("select_mask"), py::arg("chunk_elems"), py::arg("n_blocks"),
        py::arg("deadline_ms"), py::arg("decisions"), py::arg("agg_kind") = 0, py::arg("trim") = 0.0);
  m.def("twoshot_resync", &twoshot_resync);
  m.def("produced_signal_pack", &produced_signal_pack);
  m.def("produced_mark", &produced_mark);
  m.def("reduce_push", &reduce_push);
}
