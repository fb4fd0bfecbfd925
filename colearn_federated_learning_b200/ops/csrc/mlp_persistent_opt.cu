// The local optimizer instances of the persistent MLP kernel (docs/KERNELS.md §5e): variant 1's shared-memory kernel with
// the local_opt.cuh step (SGD with momentum / nesterov / weight decay, or Adam) at the end of every batch, for all five
// persistent nets, dispatched by launch_mlp_local_sgd_opt.  The template code is mlp_persistent.cu's and mlp_v1_fit.inc's,
// included here unchanged.  It has a translation unit of its own for the reason mlp_persistent_ae.cu gives: new callers of
// the shared helpers change how the compiler specialises them, and with it the SASS of the existing instances.
#define COLEARN_MLP_TEMPLATES_ONLY 1
#include "mlp_persistent.cu"   // NOLINT(bugprone-suspicious-include): the kernel templates

namespace colearn {

cudaError_t launch_mlp_local_sgd_opt(int net_kind, const ClientDesc* descs, int n_clients, SgdHyper hp, LocalOptArgs lo,
                                     cudaStream_t stream) {
  switch (net_kind) {
    case NET_FFNN: return launch_opt_n<FFNNNet>(descs, n_clients, hp, lo, stream);
    case NET_MLP64: return launch_opt_n<MLP64Net>(descs, n_clients, hp, lo, stream);
    case NET_TESTING_REMOTE: return launch_opt_n<TestingRemoteNet>(descs, n_clients, hp, lo, stream);
    case NET_AE: return launch_opt_n<AENet>(descs, n_clients, hp, lo, stream);
    case NET_FFNN_CAT: return launch_opt_n<CatNet>(descs, n_clients, hp, lo, stream);
    default: return cudaErrorInvalidValue;
  }
}

COLEARN_DEFINE_SPIN_LIMIT_SETTER(set_spin_limit_mlp_opt)

}  // namespace colearn
