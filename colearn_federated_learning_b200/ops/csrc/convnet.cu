// NHWC convolution / BatchNorm / pooling kernels around the wgmma GEMM (SURVEY K17: ResNet-18 ops).
// The arithmetic of every kernel is the host+device body in conv_ops.cuh; this file only maps bodies onto
// grids: grid-stride maps (128-bit loads/stores, one work item = 8 channels) and two-phase block reductions.
#include "colearn_kernels.h"

namespace colearn {
using namespace convops;

namespace {
constexpr int kMapThreads = 256;
inline int map_grid(long long items) {
  long long b = (items + kMapThreads - 1) / kMapThreads;
  const long long cap = 132LL * 16;            // 16 resident 256-thread CTAs per SM is already more than enough
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

// every kernel exists twice: PDL = false is the plain form, PDL = true starts with the programmatic-dependent-launch
// prologue (colearn_kernels.h) and is what COLEARN_PDL=1 launches
#define COLEARN_MAP_KERNEL(NAME, ARGS, ITEMS, BODY)                                              \
  template <bool PDL>                                                                            \
  __global__ void __launch_bounds__(kMapThreads) NAME(const ARGS a) {                           \
    if (PDL) COLEARN_PDL_PROLOGUE();                                                             \
    const long long total = ITEMS(a);                                                            \
    const long long stride = (long long)gridDim.x * blockDim.x;                                  \
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) \
      BODY(a, i);                                                                                \
  }

COLEARN_MAP_KERNEL(im2col_kernel, Im2colArgs, im2col_items, im2col_body)
COLEARN_MAP_KERNEL(col2im_kernel, Col2imArgs, col2im_items, col2im_body)
COLEARN_MAP_KERNEL(bn_apply_kernel, BnApplyArgs, bn_apply_items, bn_apply_body)
COLEARN_MAP_KERNEL(bn_bwd_kernel, BnBwdArgs, bn_bwd_items, bn_bwd_body)
COLEARN_MAP_KERNEL(maxpool_fwd_kernel, PoolArgs, maxpool_fwd_items, maxpool_fwd_body)
COLEARN_MAP_KERNEL(maxpool_bwd_kernel, PoolArgs, maxpool_bwd_items, maxpool_bwd_body)
COLEARN_MAP_KERNEL(avgpool_fwd_kernel, AvgPoolArgs, avgpool_fwd_items, avgpool_fwd_body)
COLEARN_MAP_KERNEL(avgpool_bwd_kernel, AvgPoolArgs, avgpool_bwd_items, avgpool_bwd_body)

__device__ __forceinline__ long long pack_items(const PackArgs& a) { return a.total; }
COLEARN_MAP_KERNEL(pack_kernel, PackArgs, pack_items, pack_body)
COLEARN_MAP_KERNEL(splitk_reduce_kernel, SplitKReduceArgs, splitk_reduce_items, splitk_reduce_body)

// grid = (C/64, nseg), 256 threads
template <bool PDL>
__global__ void __launch_bounds__(kBnThreads) bn_reduce_kernel(const BnReduceArgs a) {
  if (PDL) COLEARN_PDL_PROLOGUE();
  __shared__ float smem[kBnSmemFloats];
  bn_reduce_phase1(a, blockIdx.x, blockIdx.y, threadIdx.x, smem);
  __syncthreads();
  bn_reduce_phase2(a, blockIdx.x, blockIdx.y, threadIdx.x, smem);
}
template <bool PDL>
__global__ void bn_finalize_kernel(const BnFinalizeArgs a) {
  if (PDL) COLEARN_PDL_PROLOGUE();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < a.C) bn_finalize_body<false>(a, c);
}
// reduction + finalize fused: the last block of each column group (ticket counter) finalises it
template <bool PDL>
__global__ void __launch_bounds__(kBnThreads) bn_reduce_finalize_kernel(const BnFusedArgs a) {
  if (PDL) COLEARN_PDL_PROLOGUE();
  __shared__ float smem[kBnSmemFloats];
  __shared__ int s_last;
  bn_reduce_phase1(a.r, blockIdx.x, blockIdx.y, threadIdx.x, smem);
  __syncthreads();
  bn_reduce_phase2(a.r, blockIdx.x, blockIdx.y, threadIdx.x, smem);
  __threadfence();                 // partials of this block visible device-wide before the ticket
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(&a.counters[blockIdx.x], 1u) == gridDim.y - 1) ? 1 : 0;
  __syncthreads();
  if (s_last) {
    __threadfence();
    bn_fused_phase3(a, blockIdx.x, threadIdx.x);
    if (threadIdx.x == 0) a.counters[blockIdx.x] = 0;
  }
}
// plain kernel, or its PDL twin with the programmatic-launch attribute when COLEARN_PDL=1
#ifdef COLEARN_HOST_SHIM
#define COLEARN_LAUNCH1(NAME, GRID, BLOCK) (COLEARN_LAUNCH(NAME<false>, GRID, BLOCK, 0, s, a), cudaSuccess)
#else
#define COLEARN_LAUNCH1(NAME, GRID, BLOCK) launch_maybe_pdl(NAME<false>, NAME<true>, dim3(GRID), dim3(BLOCK), s, a)
#endif
}  // namespace

cudaError_t launch_im2col(const Im2colArgs& a, cudaStream_t s) {
  return COLEARN_LAUNCH1(im2col_kernel, map_grid(im2col_items(a)), kMapThreads);
}
cudaError_t launch_col2im(const Col2imArgs& a, cudaStream_t s) {
  return COLEARN_LAUNCH1(col2im_kernel, map_grid(col2im_items(a)), kMapThreads);
}
cudaError_t launch_bn_reduce(const BnReduceArgs& a, cudaStream_t s) {
  dim3 grid(a.C / kBnCols, bn_nseg(a));
  return COLEARN_LAUNCH1(bn_reduce_kernel, grid, kBnThreads);
}
cudaError_t launch_bn_reduce_finalize(const BnFusedArgs& a, cudaStream_t s) {
  dim3 grid(a.r.C / kBnCols, bn_nseg(a.r));
  return COLEARN_LAUNCH1(bn_reduce_finalize_kernel, grid, kBnThreads);
}
cudaError_t launch_bn_finalize(const BnFinalizeArgs& a, cudaStream_t s) {
  return COLEARN_LAUNCH1(bn_finalize_kernel, (a.C + 63) / 64, 64);
}
cudaError_t launch_bn_apply(const BnApplyArgs& a, cudaStream_t s) {
  return COLEARN_LAUNCH1(bn_apply_kernel, map_grid(bn_apply_items(a)), kMapThreads);
}
cudaError_t launch_bn_bwd(const BnBwdArgs& a, cudaStream_t s) {
  return COLEARN_LAUNCH1(bn_bwd_kernel, map_grid(bn_bwd_items(a)), kMapThreads);
}
cudaError_t launch_maxpool_fwd(const PoolArgs& a, cudaStream_t s) {
  return COLEARN_LAUNCH1(maxpool_fwd_kernel, map_grid(maxpool_fwd_items(a)), kMapThreads);
}
cudaError_t launch_maxpool_bwd(const PoolArgs& a, cudaStream_t s) {
  return COLEARN_LAUNCH1(maxpool_bwd_kernel, map_grid(maxpool_bwd_items(a)), kMapThreads);
}
cudaError_t launch_avgpool_fwd(const AvgPoolArgs& a, cudaStream_t s) {
  return COLEARN_LAUNCH1(avgpool_fwd_kernel, map_grid(avgpool_fwd_items(a)), kMapThreads);
}
cudaError_t launch_avgpool_bwd(const AvgPoolArgs& a, cudaStream_t s) {
  return COLEARN_LAUNCH1(avgpool_bwd_kernel, map_grid(avgpool_bwd_items(a)), kMapThreads);
}
cudaError_t launch_pack(const PackArgs& a, cudaStream_t s) {
  return COLEARN_LAUNCH1(pack_kernel, map_grid(a.total), kMapThreads);
}
cudaError_t launch_splitk_reduce(const SplitKReduceArgs& a, cudaStream_t s) {
  return COLEARN_LAUNCH1(splitk_reduce_kernel, map_grid(splitk_reduce_items(a)), kMapThreads);
}

}  // namespace colearn
