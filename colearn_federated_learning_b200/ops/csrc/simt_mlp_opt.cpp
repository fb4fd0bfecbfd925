// mlp_persistent_opt.cu (the local optimizer instances) compiled for the CPU through host_shim.h — see simt_emul.cpp
#define COLEARN_HOST_SHIM 1
#include "host_shim.h"

#include "mlp_persistent_opt.cu"   // NOLINT(bugprone-suspicious-include): the kernel source itself
