// The class-weighted instances of the persistent MLP kernel (docs/KERNELS.md §5d): variant 5, batch 1 and accumulating, for the
// FFNN and the attack-category net, dispatched by launch_mlp_local_sgd_cw.  The template code is mlp_persistent.cu's and
// mlp_v2.cuh's, included here unchanged, with the fused head's class-weight switch on.  It has a translation unit of its own for
// the reason mlp_persistent_ae.cu gives: a new caller of the non-template helpers of mlp_v2.cuh changes how the compiler
// specialises them, and with it the SASS of the unweighted instances.
#define COLEARN_MLP_TEMPLATES_ONLY 1
#include "mlp_persistent.cu"   // NOLINT(bugprone-suspicious-include): the kernel templates

namespace colearn {

cudaError_t launch_mlp_local_sgd_cw(int net_kind, const ClientDesc* descs, int n_clients, SgdHyper hp, ClassWeights cw,
                                    cudaStream_t stream) {
  if (hp.variant != 5) return cudaErrorInvalidValue;
  switch (net_kind) {
    case NET_FFNN:
      if (hp.loss == LOSS_XENT) return cudaErrorInvalidValue;   // the sigmoid head's losses: bce, sse, mse
      return v2_128b::launch2_cw<FFNNNet>(descs, n_clients, hp, cw, stream);
    case NET_FFNN_CAT:
      if (hp.loss != LOSS_XENT) return cudaErrorInvalidValue;   // the class index is the softmax head's label
      return v2_128b::launch2_cw<CatNet>(descs, n_clients, hp, cw, stream);
    default: return cudaErrorInvalidValue;
  }
}

COLEARN_DEFINE_SPIN_LIMIT_SETTER(set_spin_limit_mlp_cw)

}  // namespace colearn
