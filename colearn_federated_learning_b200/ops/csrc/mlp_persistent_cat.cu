// The attack-category FFNN's instances (CatNet, 10-50-30-10-5, softmax cross-entropy) of the persistent MLP kernels: variants
// 1, 3, 5 and 6 and the batched forward, dispatched from mlp_persistent.cu's launchers for NET_FFNN_CAT.  The template code is
// mlp_persistent.cu's and mlp_v2.cuh's, included here unchanged.  It has a translation unit of its own for the reason
// mlp_persistent_ae.cu gives: a new caller of the non-template helpers of mlp_v2.cuh changes how the compiler specialises
// them, and with it the SASS of the FFNN instances.
#define COLEARN_MLP_TEMPLATES_ONLY 1
#include "mlp_persistent.cu"   // NOLINT(bugprone-suspicious-include): the kernel templates

namespace colearn {

cudaError_t launch_mlp_local_sgd_cat(const ClientDesc* descs, int n_clients, SgdHyper hp, cudaStream_t stream) {
  switch (hp.variant) {
    case 6: return v2_128p::launch2<CatNet>(descs, n_clients, hp, stream);
    case 5: return v2_128b::launch2<CatNet>(descs, n_clients, hp, stream);
    case 3: return v2_128::launch2<CatNet>(descs, n_clients, hp, stream);
    case 1: return launch_t<CatNet>(descs, n_clients, hp, stream);
    default: return cudaErrorInvalidValue;
  }
}

int mlp_local_sgd_smem_bytes_cat(int batch_size) { return smem_bytes<CatNet>(batch_size); }

int mlp_net_num_params_cat() { return Totals<CatNet>::flat_params; }

cudaError_t launch_mlp_forward_cat(const float* theta, const float* x, float* out, int n, cudaStream_t stream) {
  return forward_t<CatNet>(theta, x, out, n, stream);
}

COLEARN_DEFINE_SPIN_LIMIT_SETTER(set_spin_limit_mlp_cat)

}  // namespace colearn
