// wgmma / TMA GEMM for sm_90a:  C[M,N] = A[M,K] . B[N,K]^T   (bf16 in, fp32 accumulate)
//
// Serves the Linear layers of the wide models (SURVEY K7/K8): forward (bias+ReLU epilogue),
// dgrad (ReLU-mask epilogue) and wgrad (fused bias-grad column sums + fused SGD update of the fp32
// master weights and refresh of the bf16 shadows W / W^T).  All three are expressed as the same
// "both operands K-major" product by keeping transposed bf16 copies that the producing epilogue
// writes for free (out_bf16_t: lanes of a warp hold 32 consecutive rows, so the transposed store is
// naturally coalesced).
//
// Fused broadcast -> GEMM (SURVEY K1): when ep.ready_flags is set, the TMA producer polls
// (ld.acquire.sys) the per-chunk ready flag of the B rows it is about to fetch — flags that the
// two-shot FedAvg kernel on a PEER GPU raises after writing the new weights over NVLink — then
// issues fence.proxy.async before the cp.async.bulk.tensor, so the first layer's GEMM starts on
// the tiles that have landed while later chunks are still in flight.
//
// Structure (persistent, 1 CTA / SM, 384 threads = 3 warpgroups):
//   warpgroup 0   : TMA producer (1 elected lane)   smem ring of kStages x {A 128x64, B BNx64} bf16, SW128
//   warpgroups 1-2: consumers, rows [0, 64) / [64, 128) of the tile: wgmma.m64nBNk16 from shared memory into
//                   registers, then the fused epilogue through a per-warpgroup fp32 staging tile (the accumulator
//                   fragment holds 2 rows x 2 columns per thread; the epilogue wants one row x 32 columns per lane)
#include "colearn_kernels.h"
#include "produced.cuh"

#include <cuda.h>
#include <cuda_bf16.h>

#include <mutex>
#include <string>
#include <unordered_map>

namespace colearn {
namespace {

constexpr int BM = 128, BK = 64;
constexpr int WG_K = 16;                           // K of one wgmma
constexpr int kConsumers = 2;                      // consumer warpgroups, 64 tile rows each
constexpr int kThreads = 128 * (1 + kConsumers);
constexpr int kMaxStages = 6;
constexpr int kEpiStride = 65;                     // fp32 staging row pitch: odd, so a warp's 32 row reads hit 32 banks
constexpr int kEpiBytes = kConsumers * 64 * kEpiStride * 4;
// Tile config.  BN = 256 halves the B-operand smem traffic per FLOP; the ring is as deep as the 227 KB of shared memory
// a block may use allows next to the staging tiles.
template <int BN_>
struct Cfg {
  static constexpr int kStages = BN_ == 256 ? 4 : 6;
  static constexpr uint32_t kStageBytesA = BM * BK * 2, kStageBytesB = BN_ * BK * 2;
  static constexpr uint32_t kStageBytes = kStageBytesA + kStageBytesB;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/ + kEpiBytes;
  static_assert(kSmemBytes <= 227 * 1024, "H100: at most 227 KB of shared memory per block");
};

std::string g_last_error;

// Opt-in limit of dynamic shared memory: operand stages + barriers + staging
inline cudaError_t configure_smem(const void* kernel, int base_bytes, int dev) {
#ifdef COLEARN_HOST_SHIM
  (void)kernel; (void)base_bytes; (void)dev;
  return cudaSuccess;
#else
  (void)dev;
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, base_bytes);
#endif
}

#ifdef COLEARN_HOST_SHIM
#include "gemm_host_model.h"   // functional CPU model of mbarrier / TMA / wgmma (tests)
#else
// ---- PTX wrappers -------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar_addr, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t"
      "}" : "=r"(done) : "r"(bar_addr), "r"(parity) : "memory");
  return done;
}
// Watchdog: a wait that lasts longer than this can only be a protocol bug (e.g. a TMA box whose byte count does not match
// the expect_tx of its stage) — trap, so that the launch fails with an error instead of hanging the GPU.
constexpr unsigned long long kMbarTimeoutNs = 20ull * 1000 * 1000 * 1000;
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  if (mbar_try_wait(addr, parity)) return;
  unsigned long long t0, t1;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  for (;;) {
    if (mbar_try_wait(addr, parity)) return;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    if (t1 - t0 > kMbarTimeoutNs) __trap();
  }
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* tmap, int c0, int c1, int c2, int c3, uint64_t* bar) {
  // 4-D tiled box (implicit-GEMM convolution: (channel, w, h, image) of an NHWC activation); coordinates may be
  // negative / past the edge, those elements are zero-filled
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
      ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_2d_mcast(void* smem_dst, const CUtensorMap* tmap, int c0, int c1, uint64_t* bar, uint16_t cta_mask) {
  // the tile lands at the same CTA-relative smem offset in every CTA of cta_mask and completes tx bytes on the
  // mbarrier at the same offset in each of them
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%2, %3}], [%4], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar)), "h"(cta_mask) : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the mbarrier at the same offset in CTA `cta_rank` of the cluster (this CTA's own rank included)
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta_rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta_rank));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// spin_wait_ge (colearn_kernels.h) without its diagnostic printf: a function call anywhere in the kernel makes ptxas
// serialise the wgmma pipeline.  Past the spin limit the launch still fails instead of hanging.
__device__ __forceinline__ void ready_wait_ge(const uint32_t* p, uint32_t want) {
  if (spin_ld_acquire_sys(p) >= want) return;
  const unsigned long long limit = g_spin_limit_ns, t0 = spin_globaltimer();
  unsigned it = 0;
  while (spin_ld_acquire_sys(p) < want) {
    __nanosleep(64);
    if (limit != 0 && (++it & 1023u) == 0 && spin_globaltimer() - t0 > limit) __trap();
  }
}
// named barrier of one consumer warpgroup (id 0 is __syncthreads)
__device__ __forceinline__ void wg_bar_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
template <int N>
__device__ __forceinline__ void set_max_regs() {
  if constexpr (N > 128) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
  else asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {   // keeps the compiler from touching d while a wgmma owns it
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64, N] += A[64, 16] . B[N, 16]^T, both operands from shared memory (TA / TB = 1: that operand is MN-major)
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, 1, 1, 1, %34, %35;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[64], uint64_t da, uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1, 1, 1, %66, %67;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[128], uint64_t da, uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, 1, 1, 1, %130, %131;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "n"(TA), "n"(TB));
}
// the fences / hints the kernels issue inline (macros, so that the statements stay exactly where they were)
#define tmap_prefetch(t) asm volatile("prefetch.tensormap [%0];" ::"l"(t) : "memory")
#define fence_mbarrier_init() asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory")
#define fence_proxy_async() asm volatile("fence.proxy.async.global;" ::: "memory")

#endif  // COLEARN_HOST_SHIM

// K-major, 128B-swizzled smem operand descriptor (sm_90 GMMA descriptor):
//   [0,14) start>>4 | [16,30) LBO>>4 (=1, ignored for swizzled K-major) | [32,46) SBO>>4 (8 rows * 128 B = 1024)
//   [62,64) layout = 1 (SWIZZLE_128B)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// MN-major, 128B-swizzled operand (canonical layout ((8,n),(8,k)):((1,LBO),(8,SBO)) in 16-byte units): the operand sits
// in shared memory the way a row-major [K rows, MN columns] global matrix lands through TMA boxes of [64 rows x 64
// columns]: inside a box, reduction row r is the 128-byte line r (8-line groups = one 1024-byte swizzle atom, SBO = 1024
// between groups); consecutive 64-column blocks are consecutive boxes (LBO = box size = 8192).
__device__ __forceinline__ uint64_t make_smem_desc_mn(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
constexpr uint32_t kMnBoxBytes = 64 * 64 * 2;                   // one [64 x 64] bf16 TMA box

// Work decomposition (tile rasterisation, split-K slices): host+device functions in conv_ops.cuh (GemmSched), shared
// with the CPU test-suite
using convops::split_kb;
using convops::work_to_tile;

struct SharedBarriers {
  uint64_t full[kMaxStages];
  uint64_t empty[kMaxStages];
};

static_assert(sizeof(SharedBarriers) <= 256, "the barriers own 256 bytes behind the operand stages");

__device__ __forceinline__ uint32_t pack2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// Fused epilogue for one 32-column chunk of one accumulator row per thread (row = m0 + 32*q + lane).
__device__ __forceinline__ void epilogue_chunk(const uint32_t (&v)[32], const GemmEpilogue& ep, int row, int col, int lane,
                                               int q, int m0, int M, int N) {
  float f[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) f[j] = __uint_as_float(v[j]);
  if (ep.bias != nullptr) {
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] += __ldg(ep.bias + col + j);
  }
  if (ep.relu) {
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] = fmaxf(f[j], 0.f);
  }
  if (ep.relu_mask != nullptr) {
    const uint4* mp = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(ep.relu_mask) + (size_t)row * N + col);
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const uint4 mv = __ldg(mp + g);
      const uint32_t w[4] = {mv.x, mv.y, mv.z, mv.w};
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        // bf16 > 0  <=>  sign bit clear and magnitude non-zero
        const uint32_t lo = w[h] & 0xFFFFu, hi = w[h] >> 16;
        if (!(lo != 0 && !(lo & 0x8000u))) f[g * 8 + h * 2] = 0.f;
        if (!(hi != 0 && !(hi & 0x8000u))) f[g * 8 + h * 2 + 1] = 0.f;
      }
    }
  }
  if (ep.addend != nullptr) {
    const uint4* ap = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(ep.addend) + (size_t)row * N + col);
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const uint4 av = __ldg(ap + g);
      const uint32_t w[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        f[g * 8 + h * 2] += __uint_as_float(w[h] << 16);              // bf16 -> fp32: the bits are the high half
        f[g * 8 + h * 2 + 1] += __uint_as_float(w[h] & 0xFFFF0000u);
      }
    }
  }
  if (ep.colsum != nullptr) {
    // bias gradient: per-(32-row block) partial column sums, plain coalesced stores (no atomics);
    // the consumer (bias_sgd_from_partials) adds the M/32 partial rows
    float mine = 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      float s = f[j];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == j) mine = s;
    }
    ep.colsum[(size_t)((m0 >> 5) + q) * N + col + lane] = mine;
  }
  if (ep.sgd_master != nullptr) {
    float4* mp = reinterpret_cast<float4*>(ep.sgd_master + (size_t)row * N + col);
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      float4 w = mp[g];
      w.x = fmaf(-ep.sgd_lr, f[g * 4 + 0], w.x); w.y = fmaf(-ep.sgd_lr, f[g * 4 + 1], w.y);
      w.z = fmaf(-ep.sgd_lr, f[g * 4 + 2], w.z); w.w = fmaf(-ep.sgd_lr, f[g * 4 + 3], w.w);
      mp[g] = w;
      f[g * 4 + 0] = w.x; f[g * 4 + 1] = w.y; f[g * 4 + 2] = w.z; f[g * 4 + 3] = w.w;  // f now holds the new weights
    }
    if (ep.sgd_shadow != nullptr) {
      uint4* sp = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(ep.sgd_shadow) + (size_t)row * N + col);
#pragma unroll
      for (int g = 0; g < 4; ++g)
        sp[g] = make_uint4(pack2(f[g * 8], f[g * 8 + 1]), pack2(f[g * 8 + 2], f[g * 8 + 3]),
                           pack2(f[g * 8 + 4], f[g * 8 + 5]), pack2(f[g * 8 + 6], f[g * 8 + 7]));
    }
    if (ep.sgd_shadow_t != nullptr) {
      __nv_bfloat16* tp = reinterpret_cast<__nv_bfloat16*>(ep.sgd_shadow_t);
#pragma unroll
      for (int j = 0; j < 32; ++j) tp[(size_t)(col + j) * M + row] = __float2bfloat16(f[j]);
    }
  } else {
    if (ep.out_f32 != nullptr) {
      float4* op = reinterpret_cast<float4*>(ep.out_f32 + (size_t)row * N + col);
#pragma unroll
      for (int g = 0; g < 8; ++g) op[g] = make_float4(f[g * 4], f[g * 4 + 1], f[g * 4 + 2], f[g * 4 + 3]);
    }
    if (ep.out_bf16 != nullptr) {
      uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(ep.out_bf16) + (size_t)row * N + col);
#pragma unroll
      for (int g = 0; g < 4; ++g)
        op[g] = make_uint4(pack2(f[g * 8], f[g * 8 + 1]), pack2(f[g * 8 + 2], f[g * 8 + 3]),
                           pack2(f[g * 8 + 4], f[g * 8 + 5]), pack2(f[g * 8 + 6], f[g * 8 + 7]));
    }
    if (ep.out_bf16_t != nullptr) {
      __nv_bfloat16* tp = reinterpret_cast<__nv_bfloat16*>(ep.out_bf16_t);
#pragma unroll
      for (int j = 0; j < 32; ++j) tp[(size_t)(col + j) * M + row] = __float2bfloat16(f[j]);
    }
  }
}

// Local-optimizer epilogue (gemm_wgmma_opt_kernel, OPT = LOCAL_OPT_SGD / LOCAL_OPT_ADAM): the accumulator is the gradient g of
// master[row, col .. col+31]; every element takes local_opt_elem (local_opt.cuh) on master, its momentum m (SGD with momentum,
// Adam) and v (Adam), all [M, N] fp32, then the bf16 shadow gets the new weights.  dW is never stored.
template <int OPT>
__device__ __forceinline__ void epilogue_opt_chunk(const uint32_t (&v)[32], const GemmEpilogue& ep, int row, int col, int N) {
  LocalOptArgs a = ep.lopt.args;
  a.kind = OPT;                                      // the optimizer branch of local_opt_elem folds at compile time
  const LocalOptStep st = ep.lopt.step;
  const bool use_m = OPT == LOCAL_OPT_ADAM || a.momentum != 0.f;
  const size_t base = (size_t)row * N + col;
  float4* wp = reinterpret_cast<float4*>(ep.sgd_master + base);
  float4* mp = reinterpret_cast<float4*>(ep.lopt.m + base);
  float4* vp = reinterpret_cast<float4*>(ep.lopt.v + base);
  uint4* sp = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(ep.sgd_shadow) + base);
#pragma unroll
  for (int h = 0; h < 4; ++h) {            // 8 columns at a time: two float4 of master / moments, one uint4 of shadow
    float f[8];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int g = h * 2 + q;
      float4 w = wp[g];
      float4 m = use_m ? mp[g] : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 s = OPT == LOCAL_OPT_ADAM ? vp[g] : make_float4(0.f, 0.f, 0.f, 0.f);
      local_opt_elem(a, st, ep.sgd_lr, w.x, __uint_as_float(v[g * 4 + 0]), m.x, s.x);
      local_opt_elem(a, st, ep.sgd_lr, w.y, __uint_as_float(v[g * 4 + 1]), m.y, s.y);
      local_opt_elem(a, st, ep.sgd_lr, w.z, __uint_as_float(v[g * 4 + 2]), m.z, s.z);
      local_opt_elem(a, st, ep.sgd_lr, w.w, __uint_as_float(v[g * 4 + 3]), m.w, s.w);
      wp[g] = w;
      if (use_m) mp[g] = m;
      if (OPT == LOCAL_OPT_ADAM) vp[g] = s;
      f[q * 4 + 0] = w.x; f[q * 4 + 1] = w.y; f[q * 4 + 2] = w.z; f[q * 4 + 3] = w.w;
    }
    if (ep.sgd_shadow != nullptr) sp[h] = make_uint4(pack2(f[0], f[1]), pack2(f[2], f[3]), pack2(f[4], f[5]), pack2(f[6], f[7]));
  }
}


// CL = 2: thread-block cluster of two CTAs working on vertically adjacent tiles (same n-block).  Each CTA fetches
// its own A tile and HALF of the shared B tile, multicasting that half into both CTAs' shared memory, which cuts
// the L2->SM operand traffic per CTA from 48 KB to 32 KB per k-block.  A stage may only be refilled when the consumers
// of BOTH CTAs are done with it: each consumer warpgroup releases the stage in its own CTA and in the peer.
// MN = true ("both operands MN-major"): A is [K, M] and B is [K, N] row-major, i.e. C = A^T B with the reduction
// running over ROWS — the conv wgrad dW[Cout, k] = sum_pixels dz[pixel, Cout] * col[pixel, k] reads dz and col as they
// are, without the two transposes a K-major kernel needs.  A stage holds 64 reduction rows; every 64-column block of
// the tile is one [64 x 64] TMA box (columns past the matrix edge are zero-filled by TMA = the Cout padding).
// BMN alone (A K-major [M, K], B [K, N] row-major): the conv dgrad dcol[pixel, k] = sum_co dz[pixel, co] * Wp[co, k]
// reads the packed weights Wp[Cout, K] as they are, so no W^T copy has to be kept in step with the SGD updates.
template <int BN, int CL, bool MN = false, bool BMN = MN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  int M, int N, int K, GemmEpilogue ep) {
  constexpr int OPT = 0;
#include "gemm_wgmma_body.inc"
}

// The wgrad dW = dz^T a of the layer-wise trainer with the local-optimizer epilogue (epilogue_opt_chunk): 1-CTA, both
// operands K-major (MN = false: the transposed copies dz^T, a^T) or both MN-major (MN = true: dz and a read in place).
// OPT = LOCAL_OPT_SGD or LOCAL_OPT_ADAM.  Same body as gemm_wgmma_kernel; only these instances read ep.lopt.
template <int BN, bool MN, int OPT_>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_opt_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                      int M, int N, int K, GemmEpilogue ep) {
  constexpr int CL = 1;
  constexpr bool BMN = MN;
  constexpr int OPT = OPT_;
#include "gemm_wgmma_body.inc"
}

// ---- host side: tensor maps ---------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode() {
#ifdef COLEARN_HOST_SHIM
  return nullptr;
#endif
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

struct MapKey {
  const void* ptr; int rows, cols, box_rows;
  bool operator==(const MapKey& o) const { return ptr == o.ptr && rows == o.rows && cols == o.cols && box_rows == o.box_rows; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    return std::hash<const void*>()(k.ptr) ^ (std::hash<int>()(k.rows) * 1000003u) ^ (std::hash<int>()(k.cols) * 10007u) ^
           (std::hash<int>()(k.box_rows) * 131u);
  }
};

bool make_tmap(const void* ptr, int rows, int cols, int box_rows, CUtensorMap* out) {
  // row-major [rows, cols] bf16; box = [box_rows rows, 64 cols] (64 bf16 = one 128-byte swizzle row)
#ifdef COLEARN_HOST_SHIM
  {
    const long long dims[2] = {cols, rows}, strides[1] = {(long long)cols * 2};
    const int box[2] = {BK, box_rows};
    shim_encode_tiled(out, ptr, 2, dims, strides, box);
    return true;
  }
#endif
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  MapKey key{ptr, rows, cols, box_rows};
  auto it = cache.find(key);
  if (it != cache.end()) { *out = it->second; return true; }
  PFN_encodeTiled enc = get_encode();
  if (enc == nullptr) { g_last_error = "cuTensorMapEncodeTiled entry point unavailable"; return false; }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMap m;
  CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { g_last_error = "cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r); return false; }
  if (cache.size() > 4096) cache.clear();
  cache[key] = m;
  *out = m;
  return true;
}

bool make_tmap_4d(const void* ptr, int n_images, int H, int W, int C, int box_images, CUtensorMap* out) {
  // NHWC bf16 activation as (c, w, h, n); box = 64 channels x whole images (SW128: one box line = 64 channels = 128 bytes)
#ifdef COLEARN_HOST_SHIM
  {
    const long long dims[4] = {C, W, H, n_images}, strides[3] = {(long long)C * 2, (long long)W * C * 2, (long long)H * W * C * 2};
    const int box[4] = {64, W, H, box_images};
    shim_encode_tiled(out, ptr, 4, dims, strides, box);
    return true;
  }
#endif
  struct Key { const void* p; int n, h, w, c, b; bool operator==(const Key& o) const { return p == o.p && n == o.n && h == o.h && w == o.w && c == o.c && b == o.b; } };
  struct KeyHash { size_t operator()(const Key& k) const {
    return std::hash<const void*>()(k.p) ^ (size_t)k.n * 1000003u ^ (size_t)k.h * 10007u ^ (size_t)k.w * 131u ^ (size_t)k.c * 31u ^ (size_t)k.b * 7u; } };
  static std::unordered_map<Key, CUtensorMap, KeyHash> cache;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  Key key{ptr, n_images, H, W, C, box_images};
  auto it = cache.find(key);
  if (it != cache.end()) { *out = it->second; return true; }
  PFN_encodeTiled enc = get_encode();
  if (enc == nullptr) { g_last_error = "cuTensorMapEncodeTiled entry point unavailable"; return false; }
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)n_images};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {64u, (cuuint32_t)W, (cuuint32_t)H, (cuuint32_t)box_images};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUtensorMap m;
  CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { g_last_error = "cuTensorMapEncodeTiled (4-d) failed with CUresult " + std::to_string((int)r); return false; }
  if (cache.size() > 4096) cache.clear();
  cache[key] = m;
  *out = m;
  return true;
}

template <int BN, int CL>
cudaError_t launch_t(const void* A, const void* B, int M, int N, int K, const GemmEpilogue& ep, cudaStream_t s) {
  using C = Cfg<BN>;
  CUtensorMap ta, tb;
  if (!make_tmap(A, M, K, BM, &ta) || !make_tmap(B, N, K, BN / CL, &tb)) return cudaErrorInvalidValue;
  static bool configured[64] = {false};
  static int num_sms[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!configured[dev & 63]) {
    cudaError_t e = configure_smem(reinterpret_cast<const void*>(gemm_wgmma_kernel<BN, CL>), C::kSmemBytes, dev);
    if (e != cudaSuccess) { g_last_error = "cudaFuncSetAttribute(smem) failed"; return e; }
    cudaDeviceGetAttribute(&num_sms[dev & 63], cudaDevAttrMultiProcessorCount, dev);
    configured[dev & 63] = true;
  }
  const int work = (M / BM / CL) * (N / BN) * ((CL == 1 && ep.split_k > 1) ? ep.split_k : 1);
  int units = num_sms[dev & 63] / CL;          // persistent: one CTA (or CTA pair) per SM (pair)
  if (ep.max_ctas > 0 && ep.max_ctas / CL < units) units = ep.max_ctas / CL;
  if (work < units) units = work;
  if (units < 1) units = 1;
#ifdef COLEARN_HOST_SHIM
  if (CL != 1) { g_last_error = "clusters are not modelled on the host"; return cudaErrorNotSupported; }
  void (*kern)(CUtensorMap, CUtensorMap, int, int, int, GemmEpilogue) = gemm_wgmma_kernel<BN, CL>;
  COLEARN_LAUNCH(kern, units * CL, kThreads, C::kSmemBytes, s, ta, tb, M, N, K, ep);
  return cudaSuccess;
#else
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(units * CL);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = C::kSmemBytes;
  cfg.stream = s;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (CL > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = CL;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  if (ep.pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, gemm_wgmma_kernel<BN, CL>, ta, tb, M, N, K, ep);
#endif
}

// plain 1-CTA launch, with the programmatic-dependent-launch attribute when ep.pdl
inline cudaError_t launch_1cta(void (*kern)(CUtensorMap, CUtensorMap, int, int, int, GemmEpilogue), int units, int smem_bytes, cudaStream_t s,
                               const CUtensorMap& ta, const CUtensorMap& tb, int M, int N, int K, const GemmEpilogue& ep) {
#ifndef COLEARN_HOST_SHIM
  if (ep.pdl) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(units);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, ta, tb, M, N, K, ep);
  }
#endif
  COLEARN_LAUNCH(kern, units, kThreads, smem_bytes, s, ta, tb, M, N, K, ep);
  return cudaGetLastError();
}

// MN-major operands: A [K, a_cols] (AMN) or [M, K]; B [b_rows >= K, N] row-major bf16, boxes of [64 rows x 64 columns]
template <int BN, bool AMN>
cudaError_t launch_mn(const void* A, int a_cols, const void* B, int b_rows, int M, int N, int K, const GemmEpilogue& ep, cudaStream_t s) {
  using C = Cfg<BN>;
  CUtensorMap ta, tb;
  if (!(AMN ? make_tmap(A, K, a_cols, 64, &ta) : make_tmap(A, M, K, BM, &ta)) || !make_tmap(B, b_rows, N, 64, &tb))
    return cudaErrorInvalidValue;
  static bool configured[64] = {false};
  static int num_sms[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!configured[dev & 63]) {
    cudaError_t e = configure_smem(reinterpret_cast<const void*>(gemm_wgmma_kernel<BN, 1, AMN, true>), C::kSmemBytes, dev);
    if (e != cudaSuccess) { g_last_error = "cudaFuncSetAttribute(smem, mn) failed"; return e; }
    cudaDeviceGetAttribute(&num_sms[dev & 63], cudaDevAttrMultiProcessorCount, dev);
    configured[dev & 63] = true;
  }
  const int work = (M / BM) * (N / BN) * (ep.split_k > 1 ? ep.split_k : 1);
  int units = num_sms[dev & 63];
  if (ep.max_ctas > 0 && ep.max_ctas < units) units = ep.max_ctas;
  if (work < units) units = work;
  if (units < 1) units = 1;
  return launch_1cta(gemm_wgmma_kernel<BN, 1, AMN, true>, units, C::kSmemBytes, s, ta, tb, M, N, K, ep);
}

// gemm_wgmma_opt_kernel: MN = false: A [M, K], B [N, K]; MN = true: A [K, a_cols], B [K, N] (as launch_mn with a_mn = 1)
template <int BN, bool MN, int OPT>
cudaError_t launch_opt_t(const void* A, int a_cols, const void* B, int M, int N, int K, const GemmEpilogue& ep, cudaStream_t s) {
  using C = Cfg<BN>;
  CUtensorMap ta, tb;
  if (!(MN ? make_tmap(A, K, a_cols, 64, &ta) && make_tmap(B, K, N, 64, &tb) : make_tmap(A, M, K, BM, &ta) && make_tmap(B, N, K, BN, &tb)))
    return cudaErrorInvalidValue;
  static bool configured[64] = {false};
  static int num_sms[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!configured[dev & 63]) {
    cudaError_t e = configure_smem(reinterpret_cast<const void*>(gemm_wgmma_opt_kernel<BN, MN, OPT>), C::kSmemBytes, dev);
    if (e != cudaSuccess) { g_last_error = "cudaFuncSetAttribute(smem, local optimizer) failed"; return e; }
    cudaDeviceGetAttribute(&num_sms[dev & 63], cudaDevAttrMultiProcessorCount, dev);
    configured[dev & 63] = true;
  }
  const int work = (M / BM) * (N / BN);
  int units = num_sms[dev & 63];
  if (ep.max_ctas > 0 && ep.max_ctas < units) units = ep.max_ctas;
  if (work < units) units = work;
  if (units < 1) units = 1;
  return launch_1cta(gemm_wgmma_opt_kernel<BN, MN, OPT>, units, C::kSmemBytes, s, ta, tb, M, N, K, ep);
}

// The local-optimizer epilogue (ep.lopt.args.kind != 0) is the fused-SGD wgrad with another update: it takes sgd_master,
// sgd_lr, sgd_shadow and the moments, and nothing else.  The tile width follows the rule of the plain launchers (so that it
// walks the tiles the fused-SGD wgrad of the same layer walks).
cudaError_t launch_opt(const void* A, bool mn, int a_cols, const void* B, int M, int N, int K, const GemmEpilogue& ep, cudaStream_t s) {
  const LocalOptArgs& o = ep.lopt.args;
  const char* why = nullptr;
  if (o.kind != LOCAL_OPT_SGD && o.kind != LOCAL_OPT_ADAM) why = "local optimizer: kind must be LOCAL_OPT_SGD or LOCAL_OPT_ADAM";
  else if (ep.split_k > 1 || ep.cluster != 0 || ep.ready_flags != nullptr || ep.produced != nullptr || ep.colsum != nullptr ||
           ep.out_f32 != nullptr || ep.out_bf16 != nullptr || ep.out_bf16_t != nullptr || ep.conv.mode != 0)
    why = "local optimizer epilogue: no split_k, cluster, ready_flags, produced, colsum, out_* or conv";
  else if (ep.bias != nullptr || ep.relu || ep.relu_mask != nullptr || ep.addend != nullptr || ep.sgd_shadow_t != nullptr)
    why = "local optimizer epilogue: no bias, relu, relu_mask, addend or sgd_shadow_t (it is the wgrad's update)";
  else if (ep.sgd_master == nullptr || ((o.kind == LOCAL_OPT_ADAM || o.momentum != 0.f) && ep.lopt.m == nullptr) ||
           (o.kind == LOCAL_OPT_ADAM && ep.lopt.v == nullptr))
    why = "local optimizer epilogue: needs sgd_master, m (momentum / Adam) and v (Adam)";
  else if ((((uintptr_t)ep.sgd_master) | ((uintptr_t)ep.lopt.m) | ((uintptr_t)ep.lopt.v) | ((uintptr_t)ep.sgd_shadow)) & 15)
    why = "local optimizer epilogue: master, m, v and shadow must be 16-byte aligned";
  else if (ep.tile_n == 256 && (N % 256))
    why = "tile_n=256 needs N%256==0";
  if (why != nullptr) { g_last_error = why; return cudaErrorInvalidValue; }
  const bool adam = o.kind == LOCAL_OPT_ADAM;
  const bool wide = (N % 256 == 0) && ep.tile_n != 128 && (ep.tile_n == 256 || (int64_t)(M / BM) * (N / 256) >= 120);
  if (mn) {
    if (wide) return adam ? launch_opt_t<256, true, LOCAL_OPT_ADAM>(A, a_cols, B, M, N, K, ep, s) : launch_opt_t<256, true, LOCAL_OPT_SGD>(A, a_cols, B, M, N, K, ep, s);
    return adam ? launch_opt_t<128, true, LOCAL_OPT_ADAM>(A, a_cols, B, M, N, K, ep, s) : launch_opt_t<128, true, LOCAL_OPT_SGD>(A, a_cols, B, M, N, K, ep, s);
  }
  if (wide) return adam ? launch_opt_t<256, false, LOCAL_OPT_ADAM>(A, 0, B, M, N, K, ep, s) : launch_opt_t<256, false, LOCAL_OPT_SGD>(A, 0, B, M, N, K, ep, s);
  return adam ? launch_opt_t<128, false, LOCAL_OPT_ADAM>(A, 0, B, M, N, K, ep, s) : launch_opt_t<128, false, LOCAL_OPT_SGD>(A, 0, B, M, N, K, ep, s);
}

}  // namespace

const char* gemm_tcgen05_last_error() { return g_last_error.c_str(); }

template <int BN, bool WGRAD, bool BMN = WGRAD>
cudaError_t launch_conv_t(const void* act, int n_images, int H, int W, const void* other, int other_rows, int other_cols,
                          int M, int N, int K, const GemmEpilogue& ep, cudaStream_t s) {
  using C = Cfg<BN>;
  CUtensorMap ta, tb;
  const int HW = H * W;
  if (WGRAD) {   // A = dz [K pixels, a_cols] MN-major boxes, B = activation boxes of 64 pixels
    if (!make_tmap(other, other_rows, other_cols, 64, &ta) || !make_tmap_4d(act, n_images, H, W, ep.conv.C, 64 / HW, &tb))
      return cudaErrorInvalidValue;
  } else {       // A = activation boxes of 128 pixels, B = K-major weights [other_rows, other_cols] (MN-major: 64-row boxes)
    if (!make_tmap_4d(act, n_images, H, W, ep.conv.C, 128 / HW, &ta) || !make_tmap(other, other_rows, other_cols, BMN ? 64 : BN, &tb))
      return cudaErrorInvalidValue;
  }
  static bool configured[64] = {false};
  static int num_sms[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!configured[dev & 63]) {
    cudaError_t e = configure_smem(reinterpret_cast<const void*>(gemm_wgmma_kernel<BN, 1, WGRAD, BMN>), C::kSmemBytes, dev);
    if (e != cudaSuccess) { g_last_error = "cudaFuncSetAttribute(smem, conv) failed"; return e; }
    cudaDeviceGetAttribute(&num_sms[dev & 63], cudaDevAttrMultiProcessorCount, dev);
    configured[dev & 63] = true;
  }
  const int work = (M / BM) * (N / BN) * (ep.split_k > 1 ? ep.split_k : 1);
  int units = num_sms[dev & 63];
  if (ep.max_ctas > 0 && ep.max_ctas < units) units = ep.max_ctas;
  if (work < units) units = work;
  if (units < 1) units = 1;
  return launch_1cta(gemm_wgmma_kernel<BN, 1, WGRAD, BMN>, units, C::kSmemBytes, s, ta, tb, M, N, K, ep);
}

cudaError_t launch_gemm_tcgen05_conv(const void* act, int n_images, int H, int W, const void* other, int other_rows, int other_cols,
                                     int M, int N, int K, const GemmEpilogue& ep_in, cudaStream_t s) {
  GemmEpilogue ep = ep_in;
  convops::ConvAddr& g = ep.conv;
  const int HW = H * W;
  // 1x1 images (the last ResNet stage at 32x32 input): with KH = KW = 2*pad + 1 only the centre tap overlaps the image, all
  // other boxes are pure padding = zeros — walk that single tap (the caller still describes the full convolution)
  const bool centre_only = g.mode == 1 && HW == 1 && g.KH == 2 * g.pad + 1 && g.KW == 2 * g.pad + 1 && g.KH * g.KW > 1 &&
                           K == g.KH * g.KW * g.C && ep.split_k <= 1;
  g.tap_lo = centre_only ? g.pad * g.KW + g.pad : 0;
  g.tap_cnt = centre_only ? 1 : g.KH * g.KW;
  if ((g.mode != 1 && g.mode != 2) || g.C <= 0 || (g.C % 64) || g.KH <= 0 || g.KW <= 0 || g.pad < 0 || g.HW != HW ||
      !(HW == 1 || HW == 4 || HW == 16 || HW == 64) || W > 256 || H > 256 || g.n_images != n_images) {
    g_last_error = "implicit conv GEMM: mode 1|2, C%64==0, H*W in {1,4,16,64}, consistent geometry";
    return cudaErrorInvalidValue;
  }
  // N % 64 for the A-operand modes: a 64-channel layer's dgrad has only 64 output columns (128x64 tile)
  if (M <= 0 || N <= 0 || K <= 0 || (M % BM) || (N % (g.mode == 1 ? 64 : 128)) || (K % BK)) {
    g_last_error = "shape must satisfy M%128==0, N%128==0 (N%64==0 with a conv A operand), K%64==0";
    return cudaErrorInvalidValue;
  }
  if ((((uintptr_t)act) | ((uintptr_t)other)) & 15) { g_last_error = "operands must be 16-byte aligned"; return cudaErrorInvalidValue; }
  if (ep.cluster != 0 || ep.ready_flags != nullptr) { g_last_error = "implicit conv GEMM has no cluster / ready-flag variant"; return cudaErrorInvalidValue; }
  if (ep.lopt.args.kind != 0) { g_last_error = "implicit conv GEMM has no local-optimizer epilogue"; return cudaErrorInvalidValue; }
  if (g.mode == 1) {
    // M = pixels (whole images per 128-row tile), K = taps * C
    if (M != n_images * HW || K != g.KH * g.KW * g.C) { g_last_error = "implicit conv GEMM (A): M = N*H*W, K = KH*KW*C"; return cudaErrorInvalidValue; }
    if (centre_only) K = g.C;
    if (g.b_mn && !g.flip) { g_last_error = "implicit conv GEMM: the MN-major weight operand is the dgrad's"; return cudaErrorInvalidValue; }
    const int need_n = (g.KH * g.KW - 1) * g.b_rows_per_tap + N;   // dgrad: last tap's block of N weight rows / columns
    if (g.flip ? (g.b_rows_per_tap <= 0 || (g.b_mn ? (other_cols < need_n || other_rows < g.C) : (other_rows < need_n || other_cols < g.C)))
               : (other_rows < N || other_cols < K)) {
      g_last_error = "implicit conv GEMM (A): weight matrix too small";
      return cudaErrorInvalidValue;
    }
  } else {
    // K = pixels, N = padded taps * C
    if (K != n_images * HW || N < g.KH * g.KW * g.C || other_rows != K || other_cols > M || (other_cols % 8)) {
      g_last_error = "implicit conv GEMM (B): K = N*H*W, N >= KH*KW*C, dz [K, a_cols <= M]";
      return cudaErrorInvalidValue;
    }
  }
  if (ep.split_k > 1) {
    if (ep.split_out == nullptr || K / BK < ep.split_k || (((uintptr_t)ep.split_out) & 15)) {
      g_last_error = "split_k needs a 16-byte aligned split_out and K/64 >= split_k";
      return cudaErrorInvalidValue;
    }
    if (ep.bias || ep.relu || ep.relu_mask || ep.out_bf16 || ep.out_f32 || ep.out_bf16_t || ep.sgd_master || ep.colsum || ep.addend) {
      g_last_error = "split_k stores raw partials: no other epilogue option may be set";
      return cudaErrorInvalidValue;
    }
  }
  if (ep.tile_n == 256 && (N % 256)) { g_last_error = "tile_n=256 needs N%256==0"; return cudaErrorInvalidValue; }
  const bool wide = (N % 256 == 0) && ep.tile_n != 128 &&
                    (ep.tile_n == 256 || ep.split_k > 1 || (int64_t)(M / BM) * (N / 256) >= 120);
  if (g.mode == 2) {
    if (wide) return launch_conv_t<256, true>(act, n_images, H, W, other, other_rows, other_cols, M, N, K, ep, s);
    return launch_conv_t<128, true>(act, n_images, H, W, other, other_rows, other_cols, M, N, K, ep, s);
  }
  if (g.b_mn) {
    if (wide) return launch_conv_t<256, false, true>(act, n_images, H, W, other, other_rows, other_cols, M, N, K, ep, s);
    if (N % 128) return launch_conv_t<64, false, true>(act, n_images, H, W, other, other_rows, other_cols, M, N, K, ep, s);
    return launch_conv_t<128, false, true>(act, n_images, H, W, other, other_rows, other_cols, M, N, K, ep, s);
  }
  if (wide) return launch_conv_t<256, false>(act, n_images, H, W, other, other_rows, other_cols, M, N, K, ep, s);
  if (N % 128) return launch_conv_t<64, false>(act, n_images, H, W, other, other_rows, other_cols, M, N, K, ep, s);
  return launch_conv_t<128, false>(act, n_images, H, W, other, other_rows, other_cols, M, N, K, ep, s);
}

// a_mn = 1: C[M, N] = A^T B for A [K, a_cols] (a_cols <= M; the missing columns count as zeros) and B [K, N];
// a_mn = 0: C[M, N] = A B   for A [M, K] and B [b_rows >= K, N] (only the first K rows are read).  All row-major bf16.
cudaError_t launch_gemm_tcgen05_mn(const void* A, int a_mn, int a_cols, const void* B, int b_rows, int M, int N, int K,
                                   const GemmEpilogue& ep, cudaStream_t s) {
  if (M <= 0 || N <= 0 || K <= 0 || (M % BM) || (N % 128) || (K % BK) || b_rows < K) {
    g_last_error = "mn-major shape must satisfy M%128==0, N%128==0, K%64==0, b_rows >= K";
    return cudaErrorInvalidValue;
  }
  if (a_mn && (a_cols <= 0 || a_cols > M || (a_cols % 8))) {
    g_last_error = "mn-major A needs 0 < a_cols <= M, a_cols%8==0";
    return cudaErrorInvalidValue;
  }
  if ((((uintptr_t)A) | ((uintptr_t)B)) & 15) { g_last_error = "operands must be 16-byte aligned"; return cudaErrorInvalidValue; }
  if (ep.cluster != 0 || ep.ready_flags != nullptr) { g_last_error = "mn-major mode has no cluster / ready-flag variant"; return cudaErrorInvalidValue; }
  if (ep.lopt.args.kind != 0) {
    if (!a_mn) { g_last_error = "local optimizer epilogue: the mn-major form is the wgrad's (a_mn = 1)"; return cudaErrorInvalidValue; }
    return launch_opt(A, true, a_cols, B, M, N, K, ep, s);
  }
  if (ep.split_k > 1) {
    if (ep.split_out == nullptr || K / BK < ep.split_k || (((uintptr_t)ep.split_out) & 15)) {
      g_last_error = "split_k needs a 16-byte aligned split_out and K/64 >= split_k";
      return cudaErrorInvalidValue;
    }
    if (ep.bias || ep.relu || ep.relu_mask || ep.out_bf16 || ep.out_f32 || ep.out_bf16_t || ep.sgd_master || ep.colsum || ep.addend) {
      g_last_error = "split_k stores raw partials: no other epilogue option may be set";
      return cudaErrorInvalidValue;
    }
  }
  if (ep.tile_n == 256 && (N % 256)) { g_last_error = "tile_n=256 needs N%256==0"; return cudaErrorInvalidValue; }
  const bool wide = (N % 256 == 0) && ep.tile_n != 128 &&
                    (ep.tile_n == 256 || ep.split_k > 1 || (int64_t)(M / BM) * (N / 256) >= 120);
  if (a_mn) {
    if (wide) return launch_mn<256, true>(A, a_cols, B, b_rows, M, N, K, ep, s);
    return launch_mn<128, true>(A, a_cols, B, b_rows, M, N, K, ep, s);
  }
  if (wide) return launch_mn<256, false>(A, a_cols, B, b_rows, M, N, K, ep, s);
  return launch_mn<128, false>(A, a_cols, B, b_rows, M, N, K, ep, s);
}

cudaError_t launch_gemm_tcgen05(const void* A, const void* B, int M, int N, int K, const GemmEpilogue& ep, cudaStream_t s) {
  if (M <= 0 || N <= 0 || K <= 0 || (M % BM) || (N % 128) || (K % BK)) {
    g_last_error = "shape must satisfy M%128==0, N%128==0, K%64==0";
    return cudaErrorInvalidValue;
  }
  if ((((uintptr_t)A) | ((uintptr_t)B)) & 15) { g_last_error = "operands must be 16-byte aligned"; return cudaErrorInvalidValue; }
  if (ep.lopt.args.kind != 0) return launch_opt(A, false, 0, B, M, N, K, ep, s);
  if (ep.produced != nullptr && (ep.sgd_master == nullptr || ep.split_k > 1)) {
    g_last_error = "produced reports come from the fused-SGD epilogue (needs sgd_master, no split_k)";
    return cudaErrorInvalidValue;
  }
  if (ep.split_k > 1) {
    // split-K: raw fp32 partials only, 1-CTA kernel; 128x256 tiles whenever N allows (half the B smem traffic per FLOP)
    if (ep.split_out == nullptr) { g_last_error = "split_k needs split_out"; return cudaErrorInvalidValue; }
    if (K / BK < ep.split_k) { g_last_error = "split_k must not exceed K/64"; return cudaErrorInvalidValue; }
    if (ep.cluster != 0 || ep.ready_flags != nullptr || ep.bias || ep.relu || ep.relu_mask || ep.out_bf16 || ep.out_f32 ||
        ep.out_bf16_t || ep.sgd_master || ep.colsum || ep.addend) {
      g_last_error = "split_k stores raw partials: no other epilogue / cluster / ready-flag option may be set";
      return cudaErrorInvalidValue;
    }
    if (((uintptr_t)ep.split_out) & 15) { g_last_error = "split_out must be 16-byte aligned"; return cudaErrorInvalidValue; }
    if (ep.tile_n == 256 && (N % 256)) { g_last_error = "tile_n=256 needs N%256==0"; return cudaErrorInvalidValue; }
    if (ep.tile_n == 256 || (ep.tile_n == 0 && N % 256 == 0)) return launch_t<256, 1>(A, B, M, N, K, ep, s);
    return launch_t<128, 1>(A, B, M, N, K, ep, s);
  }
  // BN=256 when it divides N and leaves enough tiles to fill the machine; BN=128 otherwise
  // cluster 2 (or 3, its former name for "two SMs per 256x256 tile"): pairs of CTAs on vertically adjacent 128x256
  // tiles with TMA multicast of the shared B tile; needs M%256==0 and N%256==0, opt-in
  const bool pair = ep.cluster == 2 || ep.cluster == 3;
#ifdef COLEARN_HOST_SHIM
  if (pair) { g_last_error = "clusters are GPU-only"; return cudaErrorNotSupported; }
#endif
  if (pair && ((M % (2 * BM)) || (N % 256))) { g_last_error = "cluster=2 needs M%256==0 and N%256==0"; return cudaErrorInvalidValue; }
  if (pair) return launch_t<256, 2>(A, B, M, N, K, ep, s);
  const bool wide = (N % 256 == 0) && ((int64_t)(M / BM) * (N / 256) >= 120) && ep.tile_n != 128;
  if (wide || ep.tile_n == 256) {
    if (N % 256) { g_last_error = "tile_n=256 needs N%256==0"; return cudaErrorInvalidValue; }
    return launch_t<256, 1>(A, B, M, N, K, ep, s);
  }
  return launch_t<128, 1>(A, B, M, N, K, ep, s);
}

COLEARN_DEFINE_SPIN_LIMIT_SETTER(set_spin_limit_gemm)

}  // namespace colearn
