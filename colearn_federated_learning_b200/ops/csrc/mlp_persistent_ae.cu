// The autoencoder's instances (AENet, 10-32-4-32-10) of the persistent MLP kernels: variants 1, 3, 5 and 6 and the batched
// forward, dispatched from mlp_persistent.cu's launchers for NET_AE.  The template code is mlp_persistent.cu's and
// mlp_v2.cuh's, included here unchanged.  It is compiled in a translation unit of its own because a fourth caller of the
// non-template helpers of mlp_v2.cuh (write_out_staged) changes how the compiler specialises them, and with it the SASS of
// the FFNN instances; compiled apart, every existing instance keeps its SASS.
#define COLEARN_MLP_TEMPLATES_ONLY 1
#include "mlp_persistent.cu"   // NOLINT(bugprone-suspicious-include): the kernel templates

namespace colearn {

cudaError_t launch_mlp_local_sgd_ae(const ClientDesc* descs, int n_clients, SgdHyper hp, cudaStream_t stream) {
  switch (hp.variant) {
    case 6: return v2_128p::launch2<AENet>(descs, n_clients, hp, stream);
    case 5: return v2_128b::launch2<AENet>(descs, n_clients, hp, stream);
    case 3: return v2_128::launch2<AENet>(descs, n_clients, hp, stream);
    case 1: return launch_t<AENet>(descs, n_clients, hp, stream);
    default: return cudaErrorInvalidValue;
  }
}

int mlp_local_sgd_smem_bytes_ae(int batch_size) { return smem_bytes<AENet>(batch_size); }

int mlp_net_num_params_ae() { return Totals<AENet>::flat_params; }

cudaError_t launch_mlp_forward_ae(const float* theta, const float* x, float* out, int n, cudaStream_t stream) {
  return forward_t<AENet>(theta, x, out, n, stream);
}

COLEARN_DEFINE_SPIN_LIMIT_SETTER(set_spin_limit_mlp_ae)

}  // namespace colearn
