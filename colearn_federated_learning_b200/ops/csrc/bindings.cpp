// Torch bindings for the colearn sm_90a kernels.  Only this translation unit sees torch headers.
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda_runtime.h>

#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "colearn_kernels.h"

namespace py = pybind11;
using namespace colearn;

namespace {

inline cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

inline void check(cudaError_t e, const char* what) {
  TORCH_CHECK(e == cudaSuccess, what, ": ", cudaGetErrorString(e));
}
template <class T>
inline T* ptr_of(int64_t p) { return reinterpret_cast<T*>(static_cast<uintptr_t>(p)); }

#define CHECK_CUDA_F32(t) TORCH_CHECK((t).is_cuda() && (t).scalar_type() == at::kFloat && (t).is_contiguous(), #t " must be a contiguous CUDA float32 tensor")

// ---- persistent MLP -----------------------------------------------------------------------------
py::bytes make_client_desc(int64_t x, int64_t y, int64_t perm, int64_t theta_in, int64_t theta_out,
                           int64_t loss_out, int64_t wait_flag, int64_t wait_value, int64_t signal_flag,
                           int64_t signal_value, int64_t n, int64_t perm_rows, int64_t y_dim,
                           double out_scale, int64_t delta_mode, int64_t perm_seed, int64_t perm_row0, int64_t perm_scratch) {
  ClientDesc d;
  std::memset(&d, 0, sizeof(d));
  d.x = ptr_of<const float>(x);
  d.y = ptr_of<const float>(y);
  d.perm = ptr_of<const int>(perm);
  d.theta_in = ptr_of<const float>(theta_in);
  d.theta_out = ptr_of<float>(theta_out);
  d.loss_out = ptr_of<float>(loss_out);
  d.wait_flag = ptr_of<const uint32_t>(wait_flag);
  d.signal_flag = ptr_of<uint32_t>(signal_flag);
  d.n = (int)n;
  d.perm_rows = (int)(perm_rows > 0 ? perm_rows : 1);
  d.y_dim = (int)y_dim;
  d.wait_value = (uint32_t)wait_value;
  d.signal_value = (uint32_t)signal_value;
  d.out_scale = (float)out_scale;
  d.delta_mode = (int)delta_mode;
  d.perm_seed = (uint64_t)perm_seed;
  d.perm_row0 = (int)perm_row0;
  d.perm_scratch = ptr_of<int>(perm_scratch);
  return py::bytes(reinterpret_cast<const char*>(&d), sizeof(d));
}
int64_t client_desc_size() { return (int64_t)sizeof(ClientDesc); }

// p[0:n] *= scale for a raw device pointer (the symmetric work arena)
void scale_inplace(int64_t ptr, int64_t n, double scale) {
  check(launch_scale_inplace(ptr_of<float>(ptr), (float)scale, n, cur_stream()), "scale_inplace");
}

// limit of every bounded cross-GPU flag wait on the CURRENT device (colearn_kernels.h: spin_wait_ge); 0 = wait forever
void set_spin_limit(double seconds) {
  const unsigned long long ns = seconds <= 0 ? 0ull : (unsigned long long)(seconds * 1e9);
  check(set_spin_limit_comm(ns), "set_spin_limit (comm)");
  check(set_spin_limit_mlp(ns), "set_spin_limit (mlp)");
  check(set_spin_limit_mlp_ae(ns), "set_spin_limit (mlp, autoencoder)");
  check(set_spin_limit_gemm(ns), "set_spin_limit (gemm)");
  check(preload_comm_kernels(), "preload_comm_kernels");     // same call site: once per device, before any round
}

void mlp_local_sgd(int64_t net_kind, torch::Tensor descs, int64_t desc_offset, int64_t n_clients,
                   int64_t batch_size, int64_t epochs, int64_t max_steps, int64_t loss, double lr, int64_t variant) {
  TORCH_CHECK(descs.is_cuda() && descs.scalar_type() == at::kByte && descs.is_contiguous(), "descs must be CUDA uint8");
  TORCH_CHECK((desc_offset + n_clients) * (int64_t)sizeof(ClientDesc) <= descs.numel(), "descs too small");
  c10::cuda::CUDAGuard guard(descs.device());
  SgdHyper hp;
  hp.batch_size = (int)batch_size; hp.epochs = (int)epochs; hp.max_steps = (int)max_steps;
  hp.loss = (int)loss; hp.lr = (float)lr; hp.variant = (int)variant;
  const ClientDesc* d = reinterpret_cast<const ClientDesc*>(descs.data_ptr<uint8_t>()) + desc_offset;
  check(launch_mlp_local_sgd((int)net_kind, d, (int)n_clients, hp, cur_stream()), "mlp_local_sgd launch");
}
int64_t mlp_net_params(int64_t net_kind) { return mlp_net_num_params((int)net_kind); }
int64_t mlp_smem_bytes(int64_t net_kind, int64_t batch) { return mlp_local_sgd_smem_bytes((int)net_kind, (int)batch); }

torch::Tensor mlp_forward(int64_t net_kind, torch::Tensor theta, torch::Tensor x, int64_t d_out) {
  CHECK_CUDA_F32(theta); CHECK_CUDA_F32(x);
  c10::cuda::CUDAGuard guard(x.device());
  auto out = torch::empty({x.size(0), d_out}, x.options());
  check(launch_mlp_forward((int)net_kind, theta.data_ptr<float>(), x.data_ptr<float>(), out.data_ptr<float>(),
                           (int)x.size(0), cur_stream()), "mlp_forward launch");
  return out;
}

// ---- elementwise -----------------------------------------------------------------------------------
void sgd_step(torch::Tensor p, torch::Tensor g, double lr) {
  CHECK_CUDA_F32(p);
  TORCH_CHECK(g.is_cuda() && g.is_contiguous() && g.numel() == p.numel(), "grad shape");
  c10::cuda::CUDAGuard guard(p.device());
  if (g.scalar_type() == at::kFloat)
    check(launch_sgd_step(p.data_ptr<float>(), g.data_ptr<float>(), (float)lr, p.numel(), cur_stream()), "sgd_step");
  else if (g.scalar_type() == at::kBFloat16)
    check(launch_sgd_step_bf16grad(p.data_ptr<float>(), g.data_ptr(), (float)lr, p.numel(), cur_stream()), "sgd_step_bf16");
  else
    TORCH_CHECK(false, "grad dtype must be float32 or bfloat16");
}

// Server optimizer of the FedAvg kernels (server_opt.cuh): kind 0 = plain FedAvg with server_lr (the launch the caller made
// before optimizers existed); otherwise hyper = [beta1, beta2, tau] and m / v point to the moment buffers (v: adaptive kinds).
static ServerOptArgs server_opt_args(int64_t kind, double lr, const std::vector<double>& hyper, int64_t m, int64_t v) {
  ServerOptArgs o;
  std::memset(&o, 0, sizeof(o));
  o.kind = (int)kind;
  o.lr = (float)lr;
  if (kind != SOPT_SGD) {
    TORCH_CHECK(hyper.size() == 3, "server optimizer: hyper = [beta1, beta2, tau]");
    o.beta1 = (float)hyper[0];
    o.beta2 = (float)hyper[1];
    o.tau = (float)hyper[2];
    o.m = ptr_of<float>(m);
    o.v = ptr_of<float>(v);
  }
  TORCH_CHECK(server_opt_args_ok(o), "server optimizer: unknown kind ", kind, ", or a moment buffer missing / not 16-byte aligned");
  return o;
}

// Aggregator of the FedAvg kernels (robust_agg.cuh): kind 0 = the weighted mean; 1 = median, 2 = trimmed mean (trim per end)
static AggArgs agg_args(int64_t kind, double trim) {
  AggArgs g;
  std::memset(&g, 0, sizeof(g));
  g.kind = (int)kind;
  g.trim = (float)trim;
  TORCH_CHECK(agg_args_ok(g), "aggregator: unknown kind ", kind, " or trim fraction ", trim, " outside [0, 0.5)");
  return g;
}

// The trailing block of every fused FedAvg apply binding (launch_fedavg_apply): the server optimizer with its moment buffers, the
// aggregator (kind 0 = the weighted mean, 1 = median, 2 = trimmed mean with trim per end, 3 = geomed with iters / eps, 4 =
// norm_clip with clip), agg_weights_out (CUDA fp32 [K], distance-based kinds) and the work buffer from the caching allocator on
// theta's device.  The launcher validates the aggregator and decides which ones the rows admit.
static void fedavg_apply_rows(torch::Tensor& theta, const ClientRows& rows, double server_lr, int64_t opt_kind,
                              const std::vector<double>& opt_hyper, const c10::optional<torch::Tensor>& m,
                              const c10::optional<torch::Tensor>& v, int64_t agg_kind, double trim, int64_t iters, double eps, double clip,
                              const c10::optional<torch::Tensor>& agg_weights_out, const char* what) {
  const int64_t n = theta.numel();
  auto state = [&](const c10::optional<torch::Tensor>& t, const char* name) -> int64_t {
    if (!t.has_value()) return 0;
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kFloat && t->is_contiguous() && t->numel() >= n &&
                t->device() == theta.device(), name, ": contiguous CUDA float32 with one element per parameter, on theta's device");
    return (int64_t)reinterpret_cast<uintptr_t>(t->data_ptr<float>());
  };
  const ServerOptArgs o = server_opt_args(opt_kind, server_lr, opt_hyper, state(m, "m"), state(v, "v"));
  const AggregatorArgs g{(int)agg_kind, (float)trim, (int)iters, (float)eps, (float)clip};
  ApplyWork w{nullptr, nullptr, 0};
  if (agg_weights_out.has_value()) {
    const torch::Tensor& t = *agg_weights_out;
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat && t.is_contiguous() && t.numel() == rows.k && t.device() == theta.device(),
                "agg_weights_out: contiguous CUDA float32 [K] on theta's device");
    w.weights_out = t.data_ptr<float>();
  }
  torch::Tensor scratch;
  if (const size_t bytes = fedavg_apply_work_bytes(rows, g, n)) {
    scratch = torch::empty({(int64_t)bytes}, theta.options().dtype(at::kByte));
    w.scratch = scratch.data_ptr();
  }
  check(launch_fedavg_apply(theta.data_ptr<float>(), rows, g, o, n, w, cur_stream()), what);
}
static ClientRows client_rows(int format, int64_t k, int64_t stride, const float* weights) {
  ClientRows r{};
  r.format = format;
  r.k = (int)k;
  r.stride = stride;
  r.weights = weights;
  return r;
}

// theta += step towards the aggregate of the K models (slots fp32 [K, >= P]): the server optimizer / aggregator arguments as in
// fedavg_apply_rows; the weights are not read by the coordinate-wise kinds
void fedavg_apply(torch::Tensor theta, torch::Tensor slots, torch::Tensor weights, double server_lr, int64_t opt_kind,
                  std::vector<double> opt_hyper, c10::optional<torch::Tensor> m, c10::optional<torch::Tensor> v, int64_t agg_kind,
                  double trim, int64_t iters, double eps, double clip, c10::optional<torch::Tensor> agg_weights_out) {
  CHECK_CUDA_F32(theta); CHECK_CUDA_F32(slots); CHECK_CUDA_F32(weights);
  TORCH_CHECK(slots.dim() == 2 && slots.size(1) >= theta.numel() && weights.numel() == slots.size(0), "shapes");
  c10::cuda::CUDAGuard guard(theta.device());
  ClientRows r = client_rows(ROWS_F32, slots.size(0), slots.stride(0), weights.data_ptr<float>());
  r.models = slots.data_ptr<float>();
  fedavg_apply_rows(theta, r, server_lr, opt_kind, opt_hyper, m, v, agg_kind, trim, iters, eps, clip, agg_weights_out, "fedavg_apply");
}
// Asynchronous buffered aggregation: theta += step towards theta + aggregate of the K deltas models[k] - ring[base_slot[k]]
// (models fp32 [K, >= P], ring fp32 [slots, P] contiguous, S + 2 slots under --max-staleness S; base_slot int32 [K] on the CPU:
// the launcher checks it before it launches), the new theta also stored to ring[write_slot]; the server optimizer / aggregator
// arguments as in fedavg_apply_rows.  The slots reach the device through pinned memory without a host synchronisation.
void fedavg_apply_based(torch::Tensor theta, torch::Tensor models, torch::Tensor ring, torch::Tensor base_slot, torch::Tensor weights,
                        int64_t write_slot, double server_lr, int64_t opt_kind, std::vector<double> opt_hyper, c10::optional<torch::Tensor> m,
                        c10::optional<torch::Tensor> v, int64_t agg_kind, double trim, int64_t iters, double eps, double clip,
                        c10::optional<torch::Tensor> agg_weights_out) {
  CHECK_CUDA_F32(theta); CHECK_CUDA_F32(models); CHECK_CUDA_F32(ring); CHECK_CUDA_F32(weights);
  const int64_t n = theta.numel();
  TORCH_CHECK(models.dim() == 2 && models.stride(1) == 1 && models.size(1) >= n && weights.numel() == models.size(0) &&
              models.device() == theta.device() && weights.device() == theta.device(), "models [K, >= P], weights [K] on theta's device");
  TORCH_CHECK(ring.dim() == 2 && ring.size(1) == n && ring.is_contiguous() && ring.device() == theta.device(),
              "ring: contiguous [slots, P] on theta's device");
  TORCH_CHECK(!base_slot.is_cuda() && base_slot.scalar_type() == at::kInt && base_slot.is_contiguous() && base_slot.numel() == models.size(0),
              "base_slot: CPU int32 [K]");
  c10::cuda::CUDAGuard guard(theta.device());
  const torch::Tensor base_dev = base_slot.pin_memory().to(theta.device(), /*non_blocking=*/true);
  ClientRows r = client_rows(ROWS_F32_BASED, models.size(0), models.stride(0), weights.data_ptr<float>());
  r.models = models.data_ptr<float>();
  r.ring = ring.data_ptr<float>();
  r.ring_slots = (int)ring.size(0);
  r.write_slot = (int)write_slot;
  r.base_slot = base_dev.data_ptr<int>();
  r.base_slot_host = base_slot.data_ptr<int>();
  fedavg_apply_rows(theta, r, server_lr, opt_kind, opt_hyper, m, v, agg_kind, trim, iters, eps, clip, agg_weights_out, "fedavg_apply_based");
}
// ---- uplink codec (uplink_quant.cuh) ------------------------------------------------------------------------------------------
// (payload uint8 [K, row_bytes], scales fp32 [K, ceil(P / 256)]) of models [K, P] - theta [P] with keys int32 [K] (uint32 bits);
// row_bytes = the packed codes (P bytes for bits 8, ceil(P / 2) for bits 4) rounded up to 16 bytes
std::vector<torch::Tensor> quantize_delta(torch::Tensor models, torch::Tensor theta, torch::Tensor keys, int64_t bits) {
  CHECK_CUDA_F32(models); CHECK_CUDA_F32(theta);
  TORCH_CHECK(models.dim() == 2 && models.size(1) == theta.numel() && models.device() == theta.device(), "models [K, P], theta [P], one device");
  TORCH_CHECK(keys.is_cuda() && keys.scalar_type() == at::kInt && keys.is_contiguous() && keys.numel() == models.size(0) &&
              keys.device() == theta.device(), "keys: CUDA int32 [K] on theta's device");
  TORCH_CHECK(bits == 8 || bits == 4, "bits must be 8 or 4");
  c10::cuda::CUDAGuard guard(theta.device());
  const int64_t k = models.size(0), n = theta.numel();
  const int64_t row = ((bits == 8 ? n : (n + 1) / 2) + 15) / 16 * 16;
  auto payload = torch::empty({k, row}, models.options().dtype(at::kByte));
  auto scales = torch::empty({k, (n + kUqBlock - 1) / kUqBlock}, models.options());
  check(launch_quantize_delta(models.data_ptr<float>(), models.stride(0), theta.data_ptr<float>(),
                              reinterpret_cast<const uint32_t*>(keys.data_ptr<int>()), (int)k, (int)bits, payload.data_ptr<uint8_t>(), row,
                              scales.data_ptr<float>(), n, cur_stream()), "quantize_delta");
  return {payload, scales};
}

// theta += step towards theta + aggregate of the K decoded deltas (payload uint8 [K, >= packed codes] with 16-byte aligned rows,
// scales fp32 [K, ceil(P / 256)]); the server optimizer / aggregator arguments as in fedavg_apply_rows
void fedavg_apply_quantized(torch::Tensor theta, torch::Tensor payload, torch::Tensor scales, torch::Tensor weights, int64_t bits,
                            double server_lr, int64_t opt_kind, std::vector<double> opt_hyper, c10::optional<torch::Tensor> m,
                            c10::optional<torch::Tensor> v, int64_t agg_kind, double trim, int64_t iters, double eps, double clip,
                            c10::optional<torch::Tensor> agg_weights_out) {
  CHECK_CUDA_F32(theta); CHECK_CUDA_F32(scales); CHECK_CUDA_F32(weights);
  const int64_t n = theta.numel(), k = payload.size(0);
  TORCH_CHECK(payload.is_cuda() && payload.scalar_type() == at::kByte && payload.dim() == 2 && payload.stride(1) == 1 &&
              payload.device() == theta.device(), "payload: CUDA uint8 [K, row_bytes] on theta's device");
  TORCH_CHECK(scales.dim() == 2 && scales.size(0) == k && scales.size(1) == (n + kUqBlock - 1) / kUqBlock && weights.numel() == k &&
              scales.device() == theta.device() && weights.device() == theta.device(), "scales [K, ceil(P / 256)], weights [K]");
  TORCH_CHECK(bits == 8 || bits == 4, "bits must be 8 or 4");
  c10::cuda::CUDAGuard guard(theta.device());
  ClientRows r = client_rows(bits == 8 ? ROWS_INT8 : ROWS_INT4, k, payload.stride(0), weights.data_ptr<float>());
  r.payload = payload.data_ptr<uint8_t>();
  r.scales = scales.data_ptr<float>();
  fedavg_apply_rows(theta, r, server_lr, opt_kind, opt_hyper, m, v, agg_kind, trim, iters, eps, clip, agg_weights_out,
                    "fedavg_apply_quantized");
}

// ---- top-k uplink with error feedback (uplink_topk.cuh) -----------------------------------------------------------------------
// (indices uint8 [K, E], values fp32 [K, E]) of v = (models [K, P] - theta [P]) + residual [K, P], E = ut_entries(P, topk);
// residual is overwritten with the unsent part of v
std::vector<torch::Tensor> topk_delta(torch::Tensor models, torch::Tensor theta, torch::Tensor residual, int64_t topk) {
  CHECK_CUDA_F32(models); CHECK_CUDA_F32(theta); CHECK_CUDA_F32(residual);
  TORCH_CHECK(models.dim() == 2 && models.size(1) == theta.numel() && residual.sizes() == models.sizes() &&
              models.device() == theta.device() && residual.device() == theta.device(), "models / residual [K, P], theta [P], one device");
  TORCH_CHECK(topk >= 1 && topk <= kUtMaxK, "topk must be in 1..32");
  c10::cuda::CUDAGuard guard(theta.device());
  const int64_t k = models.size(0), n = theta.numel(), e = ut_entries(n, (int)topk);
  auto indices = torch::empty({k, e}, models.options().dtype(at::kByte));
  auto values = torch::empty({k, e}, models.options());
  check(launch_topk_delta(models.data_ptr<float>(), models.stride(0), theta.data_ptr<float>(), residual.data_ptr<float>(), n, (int)k,
                          (int)topk, indices.data_ptr<uint8_t>(), values.data_ptr<float>(), e, n, cur_stream()), "topk_delta");
  return {indices, values};
}

// theta += step towards theta + the weighted sum of the K sparse deltas (indices uint8 / values fp32 [K, E(P, topk)]); the
// server optimizer / aggregator arguments as in fedavg_apply_rows (the rows admit only the mean)
void fedavg_apply_topk(torch::Tensor theta, torch::Tensor indices, torch::Tensor values, torch::Tensor weights, int64_t topk,
                       double server_lr, int64_t opt_kind, std::vector<double> opt_hyper, c10::optional<torch::Tensor> m,
                       c10::optional<torch::Tensor> v, int64_t agg_kind, double trim, int64_t iters, double eps, double clip,
                       c10::optional<torch::Tensor> agg_weights_out) {
  CHECK_CUDA_F32(theta); CHECK_CUDA_F32(values); CHECK_CUDA_F32(weights);
  const int64_t n = theta.numel(), k = indices.size(0);
  TORCH_CHECK(topk >= 1 && topk <= kUtMaxK, "topk must be in 1..32");
  TORCH_CHECK(indices.is_cuda() && indices.scalar_type() == at::kByte && indices.dim() == 2 && indices.is_contiguous() &&
              indices.size(1) == ut_entries(n, (int)topk) && values.sizes() == indices.sizes() && weights.numel() == k &&
              indices.device() == theta.device() && values.device() == theta.device() && weights.device() == theta.device(),
              "indices / values [K, E(P, topk)], weights [K], on theta's device");
  c10::cuda::CUDAGuard guard(theta.device());
  ClientRows r = client_rows(ROWS_TOPK, k, indices.size(1), weights.data_ptr<float>());
  r.indices = indices.data_ptr<uint8_t>();
  r.values = values.data_ptr<float>();
  r.topk = (int)topk;
  fedavg_apply_rows(theta, r, server_lr, opt_kind, opt_hyper, m, v, agg_kind, trim, iters, eps, clip, agg_weights_out, "fedavg_apply_topk");
}

// ---- compressed downlink (downlink.cuh) -----------------------------------------------------------------------------------------
// (payload uint8 [row_bytes], scales fp32 [ceil(P / 256)]) of theta [P] - replica [P] rounded with key (uint32 bits in an int64),
// row_bytes as in quantize_delta; replica advanced in place by the decoded codes
std::vector<torch::Tensor> downlink_quant(torch::Tensor theta, torch::Tensor replica, int64_t key, int64_t bits) {
  CHECK_CUDA_F32(theta); CHECK_CUDA_F32(replica);
  TORCH_CHECK(replica.numel() == theta.numel() && replica.device() == theta.device(), "theta / replica [P], one device");
  TORCH_CHECK(bits == 8 || bits == 4, "bits must be 8 or 4");
  c10::cuda::CUDAGuard guard(theta.device());
  const int64_t n = theta.numel();
  const int64_t row = ((bits == 8 ? n : (n + 1) / 2) + 15) / 16 * 16;
  auto payload = torch::empty({row}, theta.options().dtype(at::kByte));
  auto scales = torch::empty({(n + kUqBlock - 1) / kUqBlock}, theta.options());
  check(launch_downlink_quant(theta.data_ptr<float>(), replica.data_ptr<float>(), (uint32_t)key, (int)bits, payload.data_ptr<uint8_t>(), row,
                              scales.data_ptr<float>(), n, cur_stream()), "downlink_quant");
  return {payload, scales};
}

// (indices uint8 [E], values fp32 [E]) of v = theta [P] - replica [P], E = ut_entries(P, topk); the sent entries added into replica
std::vector<torch::Tensor> downlink_topk(torch::Tensor theta, torch::Tensor replica, int64_t topk) {
  CHECK_CUDA_F32(theta); CHECK_CUDA_F32(replica);
  TORCH_CHECK(replica.numel() == theta.numel() && replica.device() == theta.device(), "theta / replica [P], one device");
  TORCH_CHECK(topk >= 1 && topk <= kUtMaxK, "topk must be in 1..32");
  c10::cuda::CUDAGuard guard(theta.device());
  const int64_t n = theta.numel(), e = ut_entries(n, (int)topk);
  auto indices = torch::empty({e}, theta.options().dtype(at::kByte));
  auto values = torch::empty({e}, theta.options());
  check(launch_downlink_topk(theta.data_ptr<float>(), replica.data_ptr<float>(), (int)topk, indices.data_ptr<uint8_t>(),
                             values.data_ptr<float>(), n, cur_stream()), "downlink_topk");
  return {indices, values};
}

// replica [P] += the decoded int8 / int4 wire (payload uint8, 16-byte aligned, a multiple of 16 bytes covering the codes;
// scales fp32 [ceil(P / 256)], validated by the caller)
void replica_apply_quant(torch::Tensor replica, torch::Tensor payload, torch::Tensor scales, int64_t bits) {
  CHECK_CUDA_F32(replica); CHECK_CUDA_F32(scales);
  const int64_t n = replica.numel();
  TORCH_CHECK(payload.is_cuda() && payload.scalar_type() == at::kByte && payload.dim() == 1 && payload.is_contiguous() &&
              payload.device() == replica.device(), "payload: contiguous CUDA uint8 [row_bytes] on the replica's device");
  TORCH_CHECK(scales.numel() == (n + kUqBlock - 1) / kUqBlock && scales.device() == replica.device(), "scales [ceil(P / 256)]");
  c10::cuda::CUDAGuard guard(replica.device());
  check(launch_replica_apply_quant(replica.data_ptr<float>(), payload.data_ptr<uint8_t>(), payload.numel(), scales.data_ptr<float>(),
                                   (int)bits, n, cur_stream()), "replica_apply_quant");
}

// replica [P] += the top-k wire (indices uint8 / values fp32 [E(P, topk)], offsets validated by the caller)
void replica_apply_topk(torch::Tensor replica, torch::Tensor indices, torch::Tensor values, int64_t topk) {
  CHECK_CUDA_F32(replica); CHECK_CUDA_F32(values);
  const int64_t n = replica.numel();
  TORCH_CHECK(topk >= 1 && topk <= kUtMaxK, "topk must be in 1..32");
  TORCH_CHECK(indices.is_cuda() && indices.scalar_type() == at::kByte && indices.is_contiguous() &&
              indices.numel() == ut_entries(n, (int)topk) && values.numel() == indices.numel() &&
              indices.device() == replica.device() && values.device() == replica.device(),
              "indices / values [E(P, topk)] on the replica's device");
  c10::cuda::CUDAGuard guard(replica.device());
  check(launch_replica_apply_topk(replica.data_ptr<float>(), indices.data_ptr<uint8_t>(), values.data_ptr<float>(), (int)topk, n,
                                  cur_stream()), "replica_apply_topk");
}

// ---- secure aggregation (secagg.cuh) ------------------------------------------------------------------------------------------
// keys: int32 [S, 8] (the little-endian words of the 32-byte stream keys), signs: int32 [S]
static void check_secagg_streams(const torch::Tensor& keys, const torch::Tensor& signs, const torch::Tensor& like) {
  TORCH_CHECK(keys.is_cuda() && keys.scalar_type() == at::kInt && keys.is_contiguous() && keys.dim() == 2 && keys.size(1) == 8 &&
              keys.device() == like.device(), "keys: contiguous CUDA int32 [S, 8] on theta's device");
  TORCH_CHECK(signs.is_cuda() && signs.scalar_type() == at::kInt && signs.is_contiguous() && signs.numel() == keys.size(0) &&
              signs.device() == like.device(), "signs: contiguous CUDA int32 [S] on theta's device");
}

// (masked int32 [P] holding the uint32 words, counts int32 [2] = clipped / non-finite) of model [P] - theta [P]
std::vector<torch::Tensor> secagg_mask(torch::Tensor model, torch::Tensor theta, torch::Tensor keys, torch::Tensor signs, double clip,
                                       int64_t frac_bits) {
  CHECK_CUDA_F32(model); CHECK_CUDA_F32(theta);
  TORCH_CHECK(model.numel() == theta.numel() && model.device() == theta.device(), "model / theta [P], one device");
  check_secagg_streams(keys, signs, theta);
  c10::cuda::CUDAGuard guard(theta.device());
  const int64_t n = theta.numel();
  auto out = torch::empty({n}, theta.options().dtype(at::kInt));
  auto counts = torch::empty({2}, theta.options().dtype(at::kInt));
  check(launch_secagg_mask(model.data_ptr<float>(), theta.data_ptr<float>(), reinterpret_cast<const uint32_t*>(keys.data_ptr<int>()),
                           signs.data_ptr<int>(), (int)keys.size(0), (float)clip, (int)frac_bits,
                           reinterpret_cast<uint32_t*>(out.data_ptr<int>()), counts.data_ptr<int>(), n, cur_stream()), "secagg_mask");
  return {out, counts};
}

// theta += step towards theta + decode(sum of the K masked rows + the signed streams) / n_mean; masked int32 [K, >= P] (uint32
// words); the server optimizer / aggregator arguments as in fedavg_apply_rows (the rows admit only the mean)
void fedavg_apply_secagg(torch::Tensor theta, torch::Tensor masked, torch::Tensor keys, torch::Tensor signs, int64_t frac_bits, int64_t n_mean,
                         double server_lr, int64_t opt_kind, std::vector<double> opt_hyper, c10::optional<torch::Tensor> m,
                         c10::optional<torch::Tensor> v, int64_t agg_kind, double trim, int64_t iters, double eps, double clip,
                         c10::optional<torch::Tensor> agg_weights_out) {
  CHECK_CUDA_F32(theta);
  const int64_t n = theta.numel();
  TORCH_CHECK(masked.is_cuda() && masked.scalar_type() == at::kInt && masked.dim() == 2 && masked.stride(1) == 1 && masked.size(1) >= n &&
              masked.device() == theta.device(), "masked: CUDA int32 [K, >= P] with unit column stride on theta's device");
  check_secagg_streams(keys, signs, theta);
  c10::cuda::CUDAGuard guard(theta.device());
  ClientRows r = client_rows(ROWS_SECAGG, masked.size(0), masked.stride(0), nullptr);
  r.masked = reinterpret_cast<const uint32_t*>(masked.data_ptr<int>());
  r.keys = reinterpret_cast<const uint32_t*>(keys.data_ptr<int>());
  r.signs = signs.data_ptr<int>();
  r.streams = (int)keys.size(0);
  r.frac_bits = (int)frac_bits;
  r.n_mean = (int)n_mean;
  fedavg_apply_rows(theta, r, server_lr, opt_kind, opt_hyper, m, v, agg_kind, trim, iters, eps, clip, agg_weights_out, "fedavg_apply_secagg");
}

torch::Tensor fedavg_flat(torch::Tensor slots, torch::Tensor weights) {
  CHECK_CUDA_F32(slots); CHECK_CUDA_F32(weights);
  TORCH_CHECK(slots.dim() == 2 && weights.numel() == slots.size(0), "shapes");
  c10::cuda::CUDAGuard guard(slots.device());
  auto out = torch::empty({slots.size(1)}, slots.options());
  check(launch_fedavg_flat(out.data_ptr<float>(), slots.data_ptr<float>(), slots.stride(0), weights.data_ptr<float>(),
                           (int)slots.size(0), slots.size(1), cur_stream()), "fedavg_flat");
  return out;
}

std::vector<torch::Tensor> sigmoid_bce(torch::Tensor z, torch::Tensor y) {
  CHECK_CUDA_F32(z); CHECK_CUDA_F32(y);
  TORCH_CHECK(z.numel() == y.numel(), "shape");
  c10::cuda::CUDAGuard guard(z.device());
  auto dz = torch::empty_like(z);
  auto loss = torch::empty({}, z.options());
  check(launch_sigmoid_bce(z.data_ptr<float>(), y.data_ptr<float>(), dz.data_ptr<float>(), loss.data_ptr<float>(), z.numel(), cur_stream()), "sigmoid_bce");
  return {loss, dz};
}
std::vector<torch::Tensor> sse_loss(torch::Tensor out, torch::Tensor y, double scale) {
  CHECK_CUDA_F32(out); CHECK_CUDA_F32(y);
  TORCH_CHECK(out.numel() == y.numel(), "shape");
  c10::cuda::CUDAGuard guard(out.device());
  auto dz = torch::empty_like(out);
  auto loss = torch::empty({}, out.options());
  check(launch_sse(out.data_ptr<float>(), y.data_ptr<float>(), dz.data_ptr<float>(), loss.data_ptr<float>(), out.numel(), (float)scale, cur_stream()), "sse");
  return {loss, dz};
}
std::vector<torch::Tensor> softmax_xent(torch::Tensor logits, torch::Tensor labels, bool want_bf16_grad) {
  TORCH_CHECK(logits.is_cuda() && logits.is_contiguous() && logits.dim() == 2, "logits");
  TORCH_CHECK(labels.is_cuda() && labels.scalar_type() == at::kLong && labels.is_contiguous() && labels.numel() == logits.size(0), "labels");
  const bool bf16 = logits.scalar_type() == at::kBFloat16;
  TORCH_CHECK(bf16 || logits.scalar_type() == at::kFloat, "logits dtype");
  c10::cuda::CUDAGuard guard(logits.device());
  auto loss = torch::empty({}, logits.options().dtype(at::kFloat));
  torch::Tensor dl, dlb;
  if (want_bf16_grad) dlb = torch::empty(logits.sizes(), logits.options().dtype(at::kBFloat16));
  else dl = torch::empty(logits.sizes(), logits.options().dtype(at::kFloat));
  check(launch_softmax_xent(logits.data_ptr(), bf16 ? 1 : 0, labels.data_ptr<int64_t>(),
                            want_bf16_grad ? nullptr : dl.data_ptr<float>(), want_bf16_grad ? dlb.data_ptr() : nullptr,
                            loss.data_ptr<float>(), (int)logits.size(0), (int)logits.size(1), cur_stream()), "softmax_xent");
  return {loss, want_bf16_grad ? dlb : dl};
}
// Fused loss head on padded operands (see softmax_xent_head_kernel): returns the mean loss; writes dl_bf16[:rows, :cols] and db[:cols].
torch::Tensor softmax_xent_head(torch::Tensor logits, torch::Tensor labels, int64_t rows, int64_t cols, c10::optional<torch::Tensor> dl_f32,
                                c10::optional<torch::Tensor> dl_bf16, c10::optional<torch::Tensor> db) {
  TORCH_CHECK(logits.is_cuda() && logits.dim() == 2 && logits.stride(1) == 1 && rows >= 1 && rows <= logits.size(0) && cols >= 1 &&
              cols <= logits.size(1), "logits [>= rows, >= cols], unit column stride");
  const bool bf16 = logits.scalar_type() == at::kBFloat16;
  TORCH_CHECK(bf16 || logits.scalar_type() == at::kFloat, "logits dtype");
  TORCH_CHECK(labels.is_cuda() && labels.scalar_type() == at::kLong && labels.is_contiguous() && labels.numel() >= rows, "labels int64 [rows]");
  float* dlp = nullptr; int ld_dl = 0; void* dbp16 = nullptr; int ld16 = 0; float* dbp = nullptr;
  if (dl_f32.has_value()) {
    TORCH_CHECK(dl_f32->is_cuda() && dl_f32->scalar_type() == at::kFloat && dl_f32->dim() == 2 && dl_f32->stride(1) == 1 &&
                dl_f32->size(0) >= rows && dl_f32->size(1) >= cols, "dl_f32");
    dlp = dl_f32->data_ptr<float>(); ld_dl = (int)dl_f32->stride(0);
  }
  if (dl_bf16.has_value()) {
    TORCH_CHECK(dl_bf16->is_cuda() && dl_bf16->scalar_type() == at::kBFloat16 && dl_bf16->dim() == 2 && dl_bf16->stride(1) == 1 &&
                dl_bf16->size(0) >= rows && dl_bf16->size(1) >= cols, "dl_bf16");
    dbp16 = dl_bf16->data_ptr(); ld16 = (int)dl_bf16->stride(0);
  }
  if (db.has_value()) {
    TORCH_CHECK(db->is_cuda() && db->scalar_type() == at::kFloat && db->is_contiguous() && db->numel() >= cols, "db fp32 [>= cols]");
    dbp = db->data_ptr<float>();
  }
  c10::cuda::CUDAGuard guard(logits.device());
  auto loss = torch::empty({}, logits.options().dtype(at::kFloat));
  check(launch_softmax_xent_head(logits.data_ptr(), bf16 ? 1 : 0, (int)logits.stride(0), labels.data_ptr<int64_t>(), dlp, ld_dl, dbp16, ld16, dbp,
                                 loss.data_ptr<float>(), (int)rows, (int)cols, cur_stream()), "softmax_xent_head");
  return loss;
}
std::vector<torch::Tensor> eval_binary(torch::Tensor p, torch::Tensor y) {
  CHECK_CUDA_F32(p); CHECK_CUDA_F32(y);
  c10::cuda::CUDAGuard guard(p.device());
  auto loss = torch::empty({}, p.options());
  auto correct = torch::empty({}, p.options().dtype(at::kInt));
  check(launch_eval_binary(p.data_ptr<float>(), y.data_ptr<float>(), loss.data_ptr<float>(), correct.data_ptr<int>(), p.numel(), cur_stream()), "eval_binary");
  return {loss, correct};
}
// Detection-metrics summary (eval_summary.cuh): scores [N, C] / labels [N] contiguous CUDA fp32 (any 4-byte alignment),
// offsets CPU int64 [S + 1]; returns (counts int64 [S, es_row_len], loss float64 [S]), views of one output block
std::vector<torch::Tensor> eval_summary(torch::Tensor scores, torch::Tensor labels, torch::Tensor offsets, int64_t bins, double threshold,
                                        int64_t grid) {
  CHECK_CUDA_F32(scores); CHECK_CUDA_F32(labels);
  TORCH_CHECK(scores.dim() == 2 && labels.dim() == 1 && labels.size(0) == scores.size(0) && labels.device() == scores.device(),
              "scores [N, C], labels [N] on one device");
  TORCH_CHECK(!offsets.is_cuda() && offsets.scalar_type() == at::kLong && offsets.is_contiguous() && offsets.dim() == 1 && offsets.numel() >= 2 &&
              offsets.numel() - 1 <= INT32_MAX, "offsets: CPU int64 [S + 1]");
  const int C = (int)scores.size(1), S = (int)offsets.numel() - 1;
  TORCH_CHECK(eval_summary_args_ok(C, (int)bins, (float)threshold), "eval_summary: C in 1..32, bins a power of two in 2..4096 with C * 2 * bins <= 32768, "
              "threshold in [0, 1] (C = ", C, ", bins = ", bins, ", threshold = ", threshold, ")");
  std::vector<int64_t> table;
  const int64_t units = es_build_table(offsets.data_ptr<int64_t>(), S, table);
  TORCH_CHECK(units >= 0 && table[S] == scores.size(0), "offsets must rise from 0 to N");
  TORCH_CHECK(scores.size(0) <= kEsMaxRows, "eval_summary: at most 2^32 - 1 rows per launch (uint32 shared-memory counters)");
  c10::cuda::CUDAGuard guard(scores.device());
  auto dev_table = torch::from_blob(table.data(), {(int64_t)table.size()}, torch::kLong).to(scores.device());
  auto out = torch::empty({es_out_words(S, C, (int)bins, units)}, scores.options().dtype(at::kLong));
  EvalSummaryArgs a{scores.data_ptr<float>(), labels.data_ptr<float>(), dev_table.data_ptr<int64_t>(), S, units, C, (int)bins, (float)threshold,
                    out.data_ptr<int64_t>()};
  check(launch_eval_summary(a, (int)grid, cur_stream()), "eval_summary");
  const int64_t L = es_row_len(C, (int)bins);
  return {out.narrow(0, 0, S * L).view({S, L}), out.narrow(0, S * L, S).view(at::kDouble)};
}
// Reconstruction-error summary (recon_summary.cuh): xhat / x [N, D] contiguous CUDA fp32, labels [N] CUDA fp32 or none, offsets
// CPU int64 [S + 1]; alarm_bin >= 0 also writes the per-row error and alarm flag.  Returns (counts int64 [S, 2 + 2 B],
// err_sum float64 [S], err fp32 [N] and flag uint8 [N], both empty without alarm_bin).  Limits are checked before the launch.
std::vector<torch::Tensor> recon_summary(torch::Tensor xhat, torch::Tensor x, c10::optional<torch::Tensor> labels, torch::Tensor offsets,
                                         int64_t bins, int64_t alarm_bin, int64_t grid) {
  CHECK_CUDA_F32(xhat); CHECK_CUDA_F32(x);
  TORCH_CHECK(xhat.dim() == 2 && x.sizes() == xhat.sizes() && x.device() == xhat.device(), "xhat and x: [N, D] on one device");
  if (labels.has_value()) {
    CHECK_CUDA_F32((*labels));
    TORCH_CHECK(labels->dim() == 1 && labels->size(0) == x.size(0) && labels->device() == x.device(), "labels [N] on the device of x");
  }
  TORCH_CHECK(!offsets.is_cuda() && offsets.scalar_type() == at::kLong && offsets.is_contiguous() && offsets.dim() == 1 && offsets.numel() >= 2 &&
              offsets.numel() - 1 <= INT32_MAX, "offsets: CPU int64 [S + 1]");
  TORCH_CHECK(x.size(1) <= kRsMaxDim && recon_summary_args_ok((int)x.size(1), (int)bins) && bins <= kRsMaxBins,
              "recon_summary: D in 1..1024, bins a power of two in 32..4096 (D = ", x.size(1), ", bins = ", bins, ")");
  TORCH_CHECK(alarm_bin < 0 || alarm_bin <= bins, "recon_summary: the alarm bin must be in [0, bins]");
  const int S = (int)offsets.numel() - 1;
  std::vector<int64_t> table;
  const int64_t units = es_build_table(offsets.data_ptr<int64_t>(), S, table);
  TORCH_CHECK(units >= 0 && table[S] == x.size(0), "offsets must rise from 0 to N");
  TORCH_CHECK(x.size(0) <= kEsMaxRows, "recon_summary: at most 2^32 - 1 rows per launch (uint32 shared-memory counters)");
  c10::cuda::CUDAGuard guard(x.device());
  auto dev_table = torch::from_blob(table.data(), {(int64_t)table.size()}, torch::kLong).to(x.device());
  auto out = torch::empty({rs_out_words(S, (int)bins, units)}, x.options().dtype(at::kLong));
  const bool rows = alarm_bin >= 0;
  auto err = torch::empty({rows ? x.size(0) : 0}, x.options());
  auto flag = torch::empty({rows ? x.size(0) : 0}, x.options().dtype(at::kByte));
  ReconSummaryArgs a{xhat.data_ptr<float>(), x.data_ptr<float>(), labels.has_value() ? labels->data_ptr<float>() : nullptr,
                     dev_table.data_ptr<int64_t>(), S, units, (int)x.size(1), (int)bins, rows ? (int)alarm_bin : 0,
                     rows ? err.data_ptr<float>() : nullptr, rows ? flag.data_ptr<uint8_t>() : nullptr, out.data_ptr<int64_t>()};
  check(launch_recon_summary(a, (int)grid, cur_stream()), "recon_summary");
  const int64_t L = rs_row_len((int)bins);
  return {out.narrow(0, 0, S * L).view({S, L}), out.narrow(0, S * L, S).view(at::kDouble), err, flag};
}
torch::Tensor argmax_rows(torch::Tensor x) {
  CHECK_CUDA_F32(x);
  TORCH_CHECK(x.dim() == 2, "2-D");
  c10::cuda::CUDAGuard guard(x.device());
  auto out = torch::empty({x.size(0), 1}, x.options().dtype(at::kLong));
  check(launch_argmax_rows(x.data_ptr<float>(), out.data_ptr<int64_t>(), (int)x.size(0), (int)x.size(1), cur_stream()), "argmax");
  return out;
}
torch::Tensor minmax_scale(torch::Tensor x) {
  CHECK_CUDA_F32(x);
  TORCH_CHECK(x.dim() == 2, "2-D");
  c10::cuda::CUDAGuard guard(x.device());
  auto out = torch::empty_like(x);
  check(launch_minmax_scale(x.data_ptr<float>(), out.data_ptr<float>(), (int)x.size(0), (int)x.size(1), cur_stream()), "minmax");
  return out;
}
torch::Tensor feistel_permutation(int64_t n, int64_t rows, int64_t seed, torch::Device device) {
  if (device.is_cpu()) {   // the same bijection on the host (tests; CPU-side users of a kernel-generated order)
    auto out = torch::empty({rows, n}, torch::TensorOptions().dtype(at::kInt));
    const FeistelDomain dom = feistel_domain((uint32_t)n);
    int* p = out.data_ptr<int>();
    for (int64_t r = 0; r < rows; ++r)
      for (int64_t i = 0; i < n; ++i) p[r * n + i] = (int)feistel_index((uint32_t)i, (uint32_t)n, dom, (uint64_t)seed, (int)r);
    return out;
  }
  c10::cuda::CUDAGuard guard(device);
  auto out = torch::empty({rows, n}, torch::TensorOptions().dtype(at::kInt).device(device));
  check(launch_feistel_permutation(out.data_ptr<int>(), (int)n, (int)rows, (uint64_t)seed, cur_stream()), "feistel");
  return out;
}
torch::Tensor fp32_to_bf16(torch::Tensor x) {
  CHECK_CUDA_F32(x);
  c10::cuda::CUDAGuard guard(x.device());
  auto out = torch::empty(x.sizes(), x.options().dtype(at::kBFloat16));
  check(launch_fp32_to_bf16(x.data_ptr<float>(), out.data_ptr(), x.numel(), cur_stream()), "fp32_to_bf16");
  return out;
}
void fp32_to_bf16_into(int64_t src, int64_t dst, int64_t n) {
  check(launch_fp32_to_bf16(ptr_of<const float>(src), ptr_of<void>(dst), n, cur_stream()), "fp32_to_bf16");
}
torch::Tensor transpose_bf16(torch::Tensor x, c10::optional<torch::Tensor> out) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && x.dim() == 2 && x.is_contiguous(), "x must be contiguous CUDA bf16 [R,C]");
  c10::cuda::CUDAGuard guard(x.device());
  torch::Tensor o = out.has_value() ? *out : torch::empty({x.size(1), x.size(0)}, x.options());
  TORCH_CHECK(o.is_contiguous() && o.numel() == x.numel() && o.scalar_type() == at::kBFloat16, "out");
  check(launch_transpose_bf16(x.data_ptr(), o.data_ptr(), (int)x.size(0), (int)x.size(1), cur_stream()), "transpose_bf16");
  return o;
}
torch::Tensor fix_precision(torch::Tensor x, double base) {
  CHECK_CUDA_F32(x);
  c10::cuda::CUDAGuard guard(x.device());
  auto out = torch::empty(x.sizes(), x.options().dtype(at::kLong));
  check(launch_fix_precision(x.data_ptr<float>(), reinterpret_cast<long long*>(out.data_ptr<int64_t>()), x.numel(), base, cur_stream()), "fix_precision");
  return out;
}
torch::Tensor float_precision(torch::Tensor x, double base) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kLong && x.is_contiguous(), "x must be contiguous CUDA int64");
  c10::cuda::CUDAGuard guard(x.device());
  auto out = torch::empty(x.sizes(), x.options().dtype(at::kFloat));
  check(launch_float_precision(reinterpret_cast<const long long*>(x.data_ptr<int64_t>()), out.data_ptr<float>(), x.numel(), 1.0 / base, cur_stream()), "float_precision");
  return out;
}
torch::Tensor ring_matmul(torch::Tensor a, torch::Tensor b) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && a.scalar_type() == at::kLong && b.scalar_type() == at::kLong, "int64 CUDA tensors");
  TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && a.size(1) == b.size(0) && a.is_contiguous() && b.is_contiguous(), "A[M,K] B[K,N] contiguous");
  c10::cuda::CUDAGuard guard(a.device());
  auto out = torch::empty({a.size(0), b.size(1)}, a.options());
  check(launch_ring_matmul(reinterpret_cast<const long long*>(a.data_ptr<int64_t>()), reinterpret_cast<const long long*>(b.data_ptr<int64_t>()),
                           reinterpret_cast<long long*>(out.data_ptr<int64_t>()), (int)a.size(0), (int)a.size(1), (int)b.size(1), cur_stream()), "ring_matmul");
  return out;
}
torch::Tensor bias_sgd_from_partials(c10::optional<torch::Tensor> bias, torch::Tensor partials, double lr) {
  CHECK_CUDA_F32(partials);
  TORCH_CHECK(partials.dim() == 2, "partials [rows, n]");
  c10::cuda::CUDAGuard guard(partials.device());
  const int rows = (int)partials.size(0), n = (int)partials.size(1);
  auto grad = torch::empty({n}, partials.options());
  float* b = nullptr;
  int nb = n;
  if (bias.has_value()) {
    TORCH_CHECK(bias->is_cuda() && bias->scalar_type() == at::kFloat && bias->is_contiguous() && bias->numel() <= n, "bias");
    b = bias->data_ptr<float>();
    nb = (int)bias->numel();
  }
  check(launch_bias_sgd_from_partials(b, partials.data_ptr<float>(), rows, n, partials.stride(0), (float)lr, grad.data_ptr<float>(), nb, cur_stream()), "bias_sgd_from_partials");
  return grad;
}
void l2_flush(torch::Tensor buf) {
  CHECK_CUDA_F32(buf);
  c10::cuda::CUDAGuard guard(buf.device());
  check(launch_l2_flush(buf.data_ptr<float>(), buf.numel(), cur_stream()), "l2_flush");
}

// ---- comm ---------------------------------------------------------------------------------------------
void star_round(int64_t theta, int64_t slots, int64_t slot_stride, int64_t arrive_flags, int64_t arrive_epoch,
                std::vector<int64_t> peer_inbox, std::vector<int64_t> peer_bcast_flag, int64_t bcast_epoch,
                int64_t mc_inbox, int64_t select_mask, double server_lr, int64_t n, bool do_reduce, bool do_bcast,
                int64_t grid_counter, int64_t n_blocks, double timeout_ms, std::vector<double> weights, int64_t decision,
                int64_t opt_kind, std::vector<double> opt_hyper, int64_t opt_m, int64_t opt_v, int64_t agg_kind, double trim) {
  StarRoundArgs a;
  std::memset(&a, 0, sizeof(a));
  a.theta = ptr_of<float>(theta);
  a.slots = ptr_of<const float>(slots);
  a.slot_stride = slot_stride;
  a.arrive_flags = ptr_of<const uint32_t>(arrive_flags);
  a.arrive_epoch = (uint32_t)arrive_epoch;
  a.world = (int)peer_inbox.size();
  TORCH_CHECK(a.world <= 16 && peer_bcast_flag.size() == peer_inbox.size(), "world");
  for (int k = 0; k < a.world; ++k) {
    a.peer_inbox[k] = ptr_of<float>(peer_inbox[k]);
    a.peer_bcast_flag[k] = ptr_of<uint32_t>(peer_bcast_flag[k]);
  }
  a.bcast_epoch = (uint32_t)bcast_epoch;
  a.mc_inbox = ptr_of<float>(mc_inbox);
  a.select_mask = (uint32_t)select_mask;
  a.server_lr = (float)server_lr;
  a.n = n;
  a.do_reduce = do_reduce ? 1 : 0;
  a.do_bcast = do_bcast ? 1 : 0;
  a.grid_counter = ptr_of<uint32_t>(grid_counter);
  a.timeout_ns = timeout_ms > 0 ? (unsigned long long)(timeout_ms * 1e6) : 0ull;
  for (size_t k = 0; k < weights.size() && k < 16; ++k) a.weights[k] = (float)weights[k];
  a.decision = ptr_of<uint32_t>(decision);
  TORCH_CHECK(a.timeout_ns == 0 || a.decision != nullptr, "a deadline needs the decision scratch buffer");
  a.opt = server_opt_args(opt_kind, server_lr, opt_hyper, opt_m, opt_v);
  a.agg = agg_args(agg_kind, trim);
  check(launch_star_round(a, (int)n_blocks, cur_stream()), "star_round");
}

static TwoShotArgs make_twoshot_args(const std::vector<int64_t>& work, const std::vector<int64_t>& shadow, const std::vector<int64_t>& chunk_flags,
                    int64_t arrive_flags, int64_t weights, int64_t theta_prev, int64_t epoch, int64_t select_mask,
                    double server_lr, int64_t n, int64_t chunk_elems, int64_t rank,
                    const std::vector<int64_t>& peer_arrive, bool wait_all, int64_t mc_work, int64_t mc_shadow, int64_t produced,
                    double produced_timeout_s) {
  TwoShotArgs a;
  std::memset(&a, 0, sizeof(a));
  a.world = (int)work.size();
  TORCH_CHECK(a.world <= 16 && chunk_flags.size() == work.size(), "world");
  for (int k = 0; k < a.world; ++k) {
    a.work[k] = ptr_of<float>(work[k]);
    a.shadow_bf16[k] = shadow.empty() ? nullptr : ptr_of<void>(shadow[k]);
    a.chunk_flags[k] = ptr_of<uint32_t>(chunk_flags[k]);
  }
  a.arrive_flags = ptr_of<const uint32_t>(arrive_flags);
  a.weights = ptr_of<const float>(weights);
  a.theta_prev = ptr_of<float>(theta_prev);
  a.epoch = (uint32_t)epoch;
  a.select_mask = (uint32_t)select_mask;
  a.server_lr = (float)server_lr;
  a.n = n;
  a.chunk_elems = chunk_elems;
  a.rank = (int)rank;
  a.signal_arrive = peer_arrive.empty() ? 0 : 1;
  for (size_t k = 0; k < peer_arrive.size() && k < 16; ++k) a.peer_arrive[k] = ptr_of<uint32_t>(peer_arrive[k]);
  a.wait_all = wait_all ? 1 : 0;
  a.mc_work = ptr_of<float>(mc_work);
  a.mc_shadow = ptr_of<void>(mc_shadow);
  // overlapped form (fused wgrad GEMM -> FedAvg reduce): my [world, n_chunks] table of produced epochs
  a.produced = ptr_of<const uint32_t>(produced);
  a.produced_timeout_ns = produced_timeout_s > 0 ? (unsigned long long)(produced_timeout_s * 1e9) : 0ull;
  return a;
}

void twoshot_fedavg(std::vector<int64_t> work, std::vector<int64_t> shadow, std::vector<int64_t> chunk_flags,
                    int64_t arrive_flags, int64_t weights, int64_t theta_prev, int64_t epoch, int64_t select_mask,
                    double server_lr, int64_t n, int64_t chunk_elems, int64_t rank, int64_t n_blocks,
                    std::vector<int64_t> peer_arrive, bool wait_all, int64_t mc_work, int64_t mc_shadow, int64_t produced,
                    double produced_timeout_s, int64_t opt_kind, std::vector<double> opt_hyper, int64_t opt_m, int64_t opt_v,
                    int64_t agg_kind, double trim) {
  TwoShotArgs a = make_twoshot_args(work, shadow, chunk_flags, arrive_flags, weights, theta_prev, epoch, select_mask, server_lr, n,
                                    chunk_elems, rank, peer_arrive, wait_all, mc_work, mc_shadow, produced, produced_timeout_s);
  a.opt = server_opt_args(opt_kind, server_lr, opt_hyper, opt_m, opt_v);
  TORCH_CHECK(a.opt.kind == SOPT_SGD || (a.theta_prev != nullptr && a.mc_work == nullptr),
              "twoshot_fedavg: a server optimizer needs theta_prev and the P2P path (no multicast)");
  a.agg = agg_args(agg_kind, trim);
  TORCH_CHECK(a.agg.kind == AGG_MEAN || a.mc_work == nullptr, "twoshot_fedavg: a robust aggregator needs the P2P path (no multicast)");
  check(launch_twoshot_fedavg(a, (int)n_blocks, cur_stream()), "twoshot_fedavg");
}

// two-shot FedAvg with failure detection (TwoShotArgs::deadline_ns): the coordinator's arrived-set decision travels through
// every rank's decision ring, the result is also pushed into every rank's second arena
void twoshot_fedavg_deadline(std::vector<int64_t> work, std::vector<int64_t> shadow, std::vector<int64_t> chunk_flags,
                             int64_t arrive_flags, int64_t weights, int64_t theta_prev, int64_t epoch, int64_t select_mask,
                             double server_lr, int64_t n, int64_t chunk_elems, int64_t rank, int64_t n_blocks,
                             std::vector<int64_t> peer_arrive, bool wait_all, int64_t mc_work, int64_t mc_shadow,
                             double deadline_ms, std::vector<int64_t> decision, std::vector<int64_t> global_copy, int64_t agg_kind,
                             double trim) {
  TwoShotArgs a = make_twoshot_args(work, shadow, chunk_flags, arrive_flags, weights, theta_prev, epoch, select_mask, server_lr, n,
                                    chunk_elems, rank, peer_arrive, wait_all, mc_work, mc_shadow, 0, 0.0);
  TORCH_CHECK(deadline_ms > 0 && decision.size() == work.size() && global_copy.size() == work.size(),
              "deadline mode needs a decision ring and a second arena on every rank");
  a.deadline_ns = (unsigned long long)(deadline_ms * 1e6);
  a.true_weights = a.weights;
  for (int k = 0; k < a.world; ++k) {
    a.decision[k] = ptr_of<uint32_t>(decision[k]);
    a.global_copy[k] = ptr_of<float>(global_copy[k]);
  }
  a.agg = agg_args(agg_kind, trim);
  TORCH_CHECK(a.agg.kind == AGG_MEAN || a.mc_work == nullptr, "twoshot_fedavg: a robust aggregator needs the P2P path (no multicast)");
  check(launch_twoshot_fedavg(a, (int)n_blocks, cur_stream()), "twoshot_fedavg (deadline)");
}

void twoshot_resync(int64_t decision_ring, int64_t prev_epoch, int64_t rank, int64_t work, int64_t shadow, int64_t global_copy,
                    int64_t n, int64_t n_blocks) {
  check(launch_twoshot_resync(ptr_of<const uint32_t>(decision_ring), (uint32_t)prev_epoch, (int)rank, ptr_of<float>(work), ptr_of<void>(shadow),
                              ptr_of<const float>(global_copy), n, (int)n_blocks, cur_stream()), "twoshot_resync");
}

void reduce_push(int64_t slots, int64_t k, int64_t stride, int64_t n, int64_t dst, int64_t losses, int64_t loss_dst,
                 int64_t flag, int64_t value, int64_t counter, int64_t n_blocks) {
  check(launch_reduce_push(ptr_of<const float>(slots), (int)k, stride, n, ptr_of<float>(dst), ptr_of<const float>(losses),
                           ptr_of<float>(loss_dst), ptr_of<uint32_t>(flag), (uint32_t)value, ptr_of<uint32_t>(counter),
                           (int)n_blocks, cur_stream()), "reduce_push");
}
void set_flag(int64_t flag, int64_t value) { check(launch_set_flag(ptr_of<uint32_t>(flag), (uint32_t)value, cur_stream()), "set_flag"); }
void wait_flag(int64_t flag, int64_t value) { check(launch_wait_flag(ptr_of<const uint32_t>(flag), (uint32_t)value, cur_stream()), "wait_flag"); }
void wait_flags(int64_t flags, int64_t count, int64_t value) { check(launch_wait_flags(ptr_of<const uint32_t>(flags), (int)count, (uint32_t)value, cur_stream()), "wait_flags"); }
void wait_flags_dev(int64_t flags, int64_t count, int64_t value_ptr) { check(launch_wait_flags_dev(ptr_of<const uint32_t>(flags), (int)count, ptr_of<const uint32_t>(value_ptr), cur_stream()), "wait_flags_dev"); }
void signal_peers(std::vector<int64_t> flags, int64_t value) {
  PeerFlags f;
  std::memset(&f, 0, sizeof(f));
  TORCH_CHECK(flags.size() <= 16, "world");
  for (size_t k = 0; k < flags.size(); ++k) f.ptr[k] = ptr_of<uint32_t>(flags[k]);
  check(launch_signal_peers(f, (int)flags.size(), (uint32_t)value, cur_stream()), "signal_peers");
}
void p2p_copy(int64_t dst, int64_t src, int64_t n, int64_t flag, int64_t flag_value, int64_t n_blocks) {
  check(launch_p2p_copy(ptr_of<float>(dst), ptr_of<const float>(src), n, ptr_of<uint32_t>(flag), (uint32_t)flag_value, (int)n_blocks, cur_stream()), "p2p_copy");
}

// ---- symmetric memory via CUDA IPC (fallback when torch symmetric memory is unavailable) -----------------
int64_t ipc_alloc(int64_t bytes) {
  void* p = nullptr;
  check(cudaMalloc(&p, (size_t)bytes), "cudaMalloc");
  check(cudaMemset(p, 0, (size_t)bytes), "cudaMemset");
  return (int64_t)reinterpret_cast<uintptr_t>(p);
}
void ipc_free(int64_t p) { cudaFree(ptr_of<void>(p)); }
py::bytes ipc_get_handle(int64_t p) {
  cudaIpcMemHandle_t h;
  check(cudaIpcGetMemHandle(&h, ptr_of<void>(p)), "cudaIpcGetMemHandle");
  return py::bytes(reinterpret_cast<const char*>(&h), sizeof(h));
}
int64_t ipc_open_handle(py::bytes handle) {
  std::string s = handle;
  TORCH_CHECK(s.size() == sizeof(cudaIpcMemHandle_t), "bad handle size");
  cudaIpcMemHandle_t h;
  std::memcpy(&h, s.data(), sizeof(h));
  void* p = nullptr;
  check(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle");
  return (int64_t)reinterpret_cast<uintptr_t>(p);
}
void ipc_close_handle(int64_t p) { cudaIpcCloseMemHandle(ptr_of<void>(p)); }
bool can_access_peer(int64_t dev, int64_t peer) {
  int ok = 0;
  cudaDeviceCanAccessPeer(&ok, (int)dev, (int)peer);
  return ok != 0;
}
void enable_peer_access(int64_t peer) {
  cudaError_t e = cudaDeviceEnablePeerAccess((int)peer, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return; }
  check(e, "cudaDeviceEnablePeerAccess");
}
torch::Tensor tensor_from_ptr(int64_t p, int64_t numel, int64_t dtype_code, int64_t device_index) {
  at::ScalarType st = dtype_code == 0 ? at::kFloat : dtype_code == 1 ? at::kBFloat16 : dtype_code == 2 ? at::kInt : at::kByte;
  auto opts = torch::TensorOptions().dtype(st).device(torch::kCUDA, (int)device_index);
  return torch::from_blob(ptr_of<void>(p), {numel}, [](void*) {}, opts);
}

#include "produced_bindings.inc"
void produced_mark(int64_t sig, int64_t chunk_elems, int64_t lo, int64_t hi) {
  int shift = 0;
  while (((int64_t)1 << shift) < chunk_elems) ++shift;
  check(launch_produced_mark(ptr_of<const ProducedSignal>(sig), shift, lo, hi, cur_stream()), "produced_mark");
}

// ---- wgmma GEMM ------------------------------------------------------------------------------------------
void gemm_tcgen05(torch::Tensor A, torch::Tensor B, c10::optional<torch::Tensor> bias, bool relu,
                  c10::optional<torch::Tensor> relu_mask, c10::optional<torch::Tensor> out_bf16,
                  c10::optional<torch::Tensor> out_f32, c10::optional<torch::Tensor> out_bf16_t,
                  c10::optional<torch::Tensor> sgd_master, double sgd_lr, c10::optional<torch::Tensor> sgd_shadow,
                  c10::optional<torch::Tensor> sgd_shadow_t, c10::optional<torch::Tensor> colsum,
                  int64_t ready_flags, int64_t ready_epoch, int64_t ready_chunk_elems, int64_t ready_elem_offset, int64_t tile_n,
                  int64_t ready_epoch_ptr, int64_t cluster, int64_t split_k, c10::optional<torch::Tensor> split_out,
                  int64_t mn_m, bool b_kn, c10::optional<torch::Tensor> addend, std::vector<int64_t> conv,
                  std::vector<int64_t> produced) {
  TORCH_CHECK(A.is_cuda() && B.is_cuda() && A.scalar_type() == at::kBFloat16 && B.scalar_type() == at::kBFloat16, "A,B must be CUDA bf16");
  TORCH_CHECK(A.dim() == 2 && B.dim() == 2 && A.is_contiguous() && B.is_contiguous(), "A, B must be contiguous matrices");
  // mn_m > 0: "MN-major" operands A[K, a_cols], B[K, N] (C = A^T B, M = mn_m >= a_cols);
  // b_kn:     A[M, K] K-major, B[b_rows >= K, N] (C = A B[:K]);   else A[M, K], B[N, K] (C = A B^T)
  const bool mn = mn_m > 0;
  TORCH_CHECK(!(mn && b_kn), "mn_m and b_kn are exclusive");
  TORCH_CHECK(!conv.empty() || (mn ? A.size(0) == B.size(0) : (b_kn ? A.size(1) <= B.size(0) : A.size(1) == B.size(1))),
              mn ? "A[K,a_cols], B[K,N]" : (b_kn ? "A[M,K], B[>=K,N]" : "A[M,K], B[N,K]"));
  c10::cuda::CUDAGuard guard(A.device());
  // conv (implicit GEMM) = [mode, flip, C, KH, KW, pad, H, W, n_images, b_rows_per_tap, M, N, K, b_mn]: A is the NHWC activation
  // [n_images*H*W, C] read through a 4-D tensor map, B the other operand (mode 1: K-major weights; mode 2: dz [pixels, a_cols])
  const bool is_conv = !conv.empty();
  TORCH_CHECK(!is_conv || (conv.size() == 14 && !mn && !b_kn), "conv = 14 ints, exclusive with mn_m / b_kn");
  const int M = is_conv ? (int)conv[10] : (mn ? (int)mn_m : (int)A.size(0));
  const int N = is_conv ? (int)conv[11] : ((mn || b_kn) ? (int)B.size(1) : (int)B.size(0));
  const int K = is_conv ? (int)conv[12] : (mn ? (int)A.size(0) : (int)A.size(1));
  GemmEpilogue ep;
  std::memset(&ep, 0, sizeof(ep));
  auto chk = [&](const c10::optional<torch::Tensor>& t, at::ScalarType st, int64_t r, int64_t c, const char* name) -> void* {
    if (!t.has_value()) return nullptr;
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == st && t->is_contiguous(), name, ": dtype/contiguity");
    TORCH_CHECK(t->numel() == r * c, name, ": numel");
    return t->data_ptr();
  };
  ep.bias = (const float*)chk(bias, at::kFloat, 1, N, "bias");
  ep.relu = relu ? 1 : 0;
  ep.relu_mask = chk(relu_mask, at::kBFloat16, M, N, "relu_mask");
  ep.out_bf16 = chk(out_bf16, at::kBFloat16, M, N, "out_bf16");
  ep.out_f32 = (float*)chk(out_f32, at::kFloat, M, N, "out_f32");
  ep.out_bf16_t = chk(out_bf16_t, at::kBFloat16, N, M, "out_bf16_t");
  ep.sgd_master = (float*)chk(sgd_master, at::kFloat, M, N, "sgd_master");
  ep.sgd_lr = (float)sgd_lr;
  ep.sgd_shadow = chk(sgd_shadow, at::kBFloat16, M, N, "sgd_shadow");
  ep.sgd_shadow_t = chk(sgd_shadow_t, at::kBFloat16, N, M, "sgd_shadow_t");
  ep.colsum = (float*)chk(colsum, at::kFloat, M / 32, N, "colsum (partials [M/32, N])");
  ep.ready_flags = ptr_of<const uint32_t>(ready_flags);
  ep.ready_epoch = (uint32_t)ready_epoch;
  ep.ready_epoch_ptr = ptr_of<const uint32_t>(ready_epoch_ptr);
  ep.ready_chunk_elems = ready_chunk_elems > 0 ? ready_chunk_elems : 1;
  ep.ready_elem_offset = ready_elem_offset;
  ep.tile_n = (int)tile_n;
  ep.cluster = (int)cluster;
  ep.pdl = pdl_enabled() ? 1 : 0;      // programmatic dependent launch (on unless COLEARN_PDL=0)
  // produced = [ProducedSignal* (device), arena element of sgd_master[0, 0], max_ctas]: fused wgrad -> FedAvg reduce
  if (!produced.empty()) {
    TORCH_CHECK(produced.size() == 3, "produced = [signal_ptr, elem_offset, max_ctas]");
    ep.produced = ptr_of<const ProducedSignal>(produced[0]);
    ep.produced_elem_offset = produced[1];
    ep.max_ctas = (int)produced[2];
  }
  if (split_k > 1) {
    TORCH_CHECK(split_out.has_value() && split_out->is_cuda() && split_out->scalar_type() == at::kFloat && split_out->is_contiguous() &&
                split_out->numel() >= split_k * (int64_t)M * N, "split_out must be a contiguous CUDA fp32 tensor with >= split_k*M*N elements");
    ep.split_k = (int)split_k;
    ep.split_out = split_out->data_ptr<float>();
  }
  ep.addend = chk(addend, at::kBFloat16, M, N, "addend");
  if (is_conv) {
    convops::ConvAddr& g = ep.conv;
    g.mode = (int)conv[0]; g.flip = (int)conv[1]; g.C = (int)conv[2]; g.KH = (int)conv[3]; g.KW = (int)conv[4]; g.pad = (int)conv[5];
    const int H = (int)conv[6], W = (int)conv[7];
    g.HW = H * W; g.n_images = (int)conv[8]; g.b_rows_per_tap = (int)conv[9]; g.b_mn = (int)conv[13];
    TORCH_CHECK(A.numel() == (int64_t)g.n_images * H * W * g.C, "activation must be [n_images*H*W, C]");
    static const int dbg_lbo = std::getenv("COLEARN_UMMA_MN_LBO") ? std::atoi(std::getenv("COLEARN_UMMA_MN_LBO")) : 0;
    static const int dbg_sbo = std::getenv("COLEARN_UMMA_MN_SBO") ? std::atoi(std::getenv("COLEARN_UMMA_MN_SBO")) : 0;
    ep.mn_lbo = dbg_lbo;
    ep.mn_sbo = dbg_sbo;
    cudaError_t e = launch_gemm_tcgen05_conv(A.data_ptr(), g.n_images, H, W, B.data_ptr(), (int)B.size(0), (int)B.size(1), M, N, K, ep, cur_stream());
    TORCH_CHECK(e == cudaSuccess, "gemm_tcgen05 (implicit conv): ", cudaGetErrorString(e), " (", gemm_tcgen05_last_error(), ")");
    return;
  }
  if (mn || b_kn) {
    static const int dbg_lbo = std::getenv("COLEARN_UMMA_MN_LBO") ? std::atoi(std::getenv("COLEARN_UMMA_MN_LBO")) : 0;
    static const int dbg_sbo = std::getenv("COLEARN_UMMA_MN_SBO") ? std::atoi(std::getenv("COLEARN_UMMA_MN_SBO")) : 0;
    ep.mn_lbo = dbg_lbo;
    ep.mn_sbo = dbg_sbo;
    cudaError_t e = launch_gemm_tcgen05_mn(A.data_ptr(), mn ? 1 : 0, (int)A.size(1), B.data_ptr(), (int)B.size(0), M, N, K, ep, cur_stream());
    TORCH_CHECK(e == cudaSuccess, "gemm_tcgen05 (mn-major): ", cudaGetErrorString(e), " (", gemm_tcgen05_last_error(), ")");
    return;
  }
  cudaError_t e = launch_gemm_tcgen05(A.data_ptr(), B.data_ptr(), M, N, K, ep, cur_stream());
  TORCH_CHECK(e == cudaSuccess, "gemm_tcgen05: ", cudaGetErrorString(e), " (", gemm_tcgen05_last_error(), ")");
}

// ---- NHWC conv / BatchNorm / pooling (convnet.cu); wrappers shared with the host emulator ------------------
struct ConvCudaExec {
  static constexpr bool kCuda = true;
  static void im2col(const convops::Im2colArgs& a) { check(launch_im2col(a, cur_stream()), "im2col"); }
  static void col2im(const convops::Col2imArgs& a) { check(launch_col2im(a, cur_stream()), "col2im"); }
  static void bn_reduce(const convops::BnReduceArgs& a) { check(launch_bn_reduce(a, cur_stream()), "bn_reduce"); }
  static void bn_finalize(const convops::BnFinalizeArgs& a) { check(launch_bn_finalize(a, cur_stream()), "bn_finalize"); }
  static void bn_reduce_finalize(const convops::BnFusedArgs& a) { check(launch_bn_reduce_finalize(a, cur_stream()), "bn_reduce_finalize"); }
  static void bn_apply(const convops::BnApplyArgs& a) { check(launch_bn_apply(a, cur_stream()), "bn_apply"); }
  static void bn_bwd(const convops::BnBwdArgs& a) { check(launch_bn_bwd(a, cur_stream()), "bn_bwd"); }
  static void maxpool_fwd(const convops::PoolArgs& a) { check(launch_maxpool_fwd(a, cur_stream()), "maxpool_fwd"); }
  static void maxpool_bwd(const convops::PoolArgs& a) { check(launch_maxpool_bwd(a, cur_stream()), "maxpool_bwd"); }
  static void avgpool_fwd(const convops::AvgPoolArgs& a) { check(launch_avgpool_fwd(a, cur_stream()), "avgpool_fwd"); }
  static void avgpool_bwd(const convops::AvgPoolArgs& a) { check(launch_avgpool_bwd(a, cur_stream()), "avgpool_bwd"); }
  static void pack(const convops::PackArgs& a) { check(launch_pack(a, cur_stream()), "pack"); }
  static void splitk_reduce(const convops::SplitKReduceArgs& a) { check(launch_splitk_reduce(a, cur_stream()), "splitk_reduce"); }
};

}  // namespace

#include "conv_bindings.inc"

namespace py = pybind11;

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "colearn_federated_learning_b200 sm_90a kernels";
  m.def("make_client_desc", &make_client_desc);
  m.def("set_spin_limit", &set_spin_limit);
  m.def("scale_inplace", &scale_inplace);
  m.def("client_desc_size", &client_desc_size);
  m.def("mlp_local_sgd", &mlp_local_sgd);
  m.def("mlp_net_params", &mlp_net_params);
  m.def("mlp_smem_bytes", &mlp_smem_bytes);
  m.def("mlp_forward", &mlp_forward);
  m.def("sgd_step", &sgd_step);
  // trailing server-optimizer arguments (server_opt.cuh) default to plain FedAvg: the shorter positional calls keep working
  // trailing aggregator arguments (robust_agg.cuh, distance_agg.cuh) default to the weighted mean
  m.def("fedavg_apply", &fedavg_apply, py::arg("theta"), py::arg("slots"), py::arg("weights"), py::arg("server_lr"), py::arg("opt_kind") = 0,
        py::arg("opt_hyper") = std::vector<double>{}, py::arg("m") = py::none(), py::arg("v") = py::none(), py::arg("agg_kind") = 0,
        py::arg("trim") = 0.0, py::arg("iters") = 3,
        py::arg("eps") = 1e-6, py::arg("clip") = 0.0, py::arg("agg_weights_out") = py::none());
  m.def("fedavg_apply_based", &fedavg_apply_based, py::arg("theta"), py::arg("models"), py::arg("ring"), py::arg("base_slot"),
        py::arg("weights"), py::arg("write_slot"), py::arg("server_lr"), py::arg("opt_kind") = 0,
        py::arg("opt_hyper") = std::vector<double>{}, py::arg("m") = py::none(), py::arg("v") = py::none(), py::arg("agg_kind") = 0,
        py::arg("trim") = 0.0, py::arg("iters") = 3, py::arg("eps") = 1e-6, py::arg("clip") = 0.0, py::arg("agg_weights_out") = py::none());
  m.def("topk_delta", &topk_delta);
  m.def("fedavg_apply_topk", &fedavg_apply_topk, py::arg("theta"), py::arg("indices"), py::arg("values"), py::arg("weights"),
        py::arg("topk"), py::arg("server_lr"), py::arg("opt_kind") = 0, py::arg("opt_hyper") = std::vector<double>{},
        py::arg("m") = py::none(), py::arg("v") = py::none(), py::arg("agg_kind") = 0, py::arg("trim") = 0.0, py::arg("iters") = 3,
        py::arg("eps") = 1e-6, py::arg("clip") = 0.0, py::arg("agg_weights_out") = py::none());
  m.def("downlink_quant", &downlink_quant);
  m.def("downlink_topk", &downlink_topk);
  m.def("replica_apply_quant", &replica_apply_quant);
  m.def("replica_apply_topk", &replica_apply_topk);
  m.def("quantize_delta", &quantize_delta);
  m.def("fedavg_apply_quantized", &fedavg_apply_quantized, py::arg("theta"), py::arg("payload"), py::arg("scales"), py::arg("weights"),
        py::arg("bits"), py::arg("server_lr"), py::arg("opt_kind") = 0, py::arg("opt_hyper") = std::vector<double>{},
        py::arg("m") = py::none(), py::arg("v") = py::none(), py::arg("agg_kind") = 0, py::arg("trim") = 0.0, py::arg("iters") = 3, py::arg("eps") = 1e-6,
        py::arg("clip") = 0.0, py::arg("agg_weights_out") = py::none());
  m.def("secagg_mask", &secagg_mask);
  m.def("fedavg_apply_secagg", &fedavg_apply_secagg, py::arg("theta"), py::arg("masked"), py::arg("keys"), py::arg("signs"),
        py::arg("frac_bits"), py::arg("n_mean"), py::arg("server_lr"), py::arg("opt_kind") = 0,
        py::arg("opt_hyper") = std::vector<double>{}, py::arg("m") = py::none(), py::arg("v") = py::none(), py::arg("agg_kind") = 0,
        py::arg("trim") = 0.0, py::arg("iters") = 3, py::arg("eps") = 1e-6, py::arg("clip") = 0.0, py::arg("agg_weights_out") = py::none());
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
  m.def("fp32_to_bf16", &fp32_to_bf16);
  m.def("fp32_to_bf16_into", &fp32_to_bf16_into);
  m.def("l2_flush", &l2_flush);
  m.def("bias_sgd_from_partials", &bias_sgd_from_partials);
  m.def("fix_precision", &fix_precision);
  m.def("float_precision", &float_precision);
  m.def("ring_matmul", &ring_matmul);
  m.def("transpose_bf16", &transpose_bf16);
  m.def("star_round", &star_round, py::arg("theta"), py::arg("slots"), py::arg("slot_stride"), py::arg("arrive_flags"), py::arg("arrive_epoch"),
        py::arg("peer_inbox"), py::arg("peer_bcast_flag"), py::arg("bcast_epoch"), py::arg("mc_inbox"), py::arg("select_mask"),
        py::arg("server_lr"), py::arg("n"), py::arg("do_reduce"), py::arg("do_bcast"), py::arg("grid_counter"), py::arg("n_blocks"),
        py::arg("timeout_ms"), py::arg("weights"), py::arg("decision"), py::arg("opt_kind") = 0, py::arg("opt_hyper") = std::vector<double>{},
        py::arg("opt_m") = 0, py::arg("opt_v") = 0, py::arg("agg_kind") = 0, py::arg("trim") = 0.0);
  m.def("twoshot_fedavg", &twoshot_fedavg, py::arg("work"), py::arg("shadow"), py::arg("chunk_flags"), py::arg("arrive_flags"), py::arg("weights"),
        py::arg("theta_prev"), py::arg("epoch"), py::arg("select_mask"), py::arg("server_lr"), py::arg("n"), py::arg("chunk_elems"),
        py::arg("rank"), py::arg("n_blocks"), py::arg("peer_arrive"), py::arg("wait_all"), py::arg("mc_work"), py::arg("mc_shadow"),
        py::arg("produced"), py::arg("produced_timeout_s"), py::arg("opt_kind") = 0, py::arg("opt_hyper") = std::vector<double>{},
        py::arg("opt_m") = 0, py::arg("opt_v") = 0, py::arg("agg_kind") = 0, py::arg("trim") = 0.0);
  m.def("twoshot_fedavg_deadline", &twoshot_fedavg_deadline, py::arg("work"), py::arg("shadow"), py::arg("chunk_flags"), py::arg("arrive_flags"),
        py::arg("weights"), py::arg("theta_prev"), py::arg("epoch"), py::arg("select_mask"), py::arg("server_lr"), py::arg("n"),
        py::arg("chunk_elems"), py::arg("rank"), py::arg("n_blocks"), py::arg("peer_arrive"), py::arg("wait_all"), py::arg("mc_work"),
        py::arg("mc_shadow"), py::arg("deadline_ms"), py::arg("decision"), py::arg("global_copy"), py::arg("agg_kind") = 0, py::arg("trim") = 0.0);
  m.def("twoshot_resync", &twoshot_resync);
  m.def("produced_signal_pack", &produced_signal_pack);
  m.def("produced_mark", &produced_mark);
  m.def("reduce_push", &reduce_push);
  m.def("set_flag", &set_flag);
  m.def("wait_flag", &wait_flag);
  m.def("wait_flags", &wait_flags);
  m.def("wait_flags_dev", &wait_flags_dev);
  m.def("signal_peers", &signal_peers);
  m.def("p2p_copy", &p2p_copy);
  m.def("ipc_alloc", &ipc_alloc);
  m.def("ipc_free", &ipc_free);
  m.def("ipc_get_handle", &ipc_get_handle);
  m.def("ipc_open_handle", &ipc_open_handle);
  m.def("ipc_close_handle", &ipc_close_handle);
  m.def("can_access_peer", &can_access_peer);
  m.def("enable_peer_access", &enable_peer_access);
  m.def("tensor_from_ptr", &tensor_from_ptr);
  m.def("gemm_tcgen05", &gemm_tcgen05);
  convbind::register_ops<ConvCudaExec>(m);
}
