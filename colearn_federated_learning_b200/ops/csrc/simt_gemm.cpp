// gemm_wgmma.cu compiled for the CPU through host_shim.h + gemm_host_model.h — see simt_emul.cpp
#define COLEARN_HOST_SHIM 1
#include "host_shim.h"

#include "gemm_wgmma.cu"   // NOLINT(bugprone-suspicious-include): the kernel source itself
