// Functional CPU model of the Hopper machinery gemm_wgmma.cu is written against — mbarrier (arrival + transaction
// counts, phase parity), TMA tiled loads (2-D / 4-D boxes, SWIZZLE_128B, zero fill outside the tensor) and wgmma reading
// shared memory through GMMA descriptors (K-major and MN-major canonical layouts, the 128-byte XOR swizzle) into the
// accumulator fragment of each thread — so that the kernel SOURCE runs in the CPU test-suite through host_shim.h (one OS
// thread per CUDA thread).  It is a model of the programming interface as documented (PTX ISA: wgmma matrix descriptors
// and the m64nNk16 fp32 accumulator fragment; CUTLASS cute/arch/mma_sm90_desc.hpp), not of the hardware: what it proves
// is that the kernel's pipelines, barrier phases, work decomposition, split-K, descriptor arithmetic, TMA coordinates,
// fragment-to-row mapping and epilogues are consistent with that interface and produce the right numbers.  Asynchronous
// units (TMA, tensor core) execute synchronously at issue.
//
// Included by gemm_wgmma.cu INSTEAD of its PTX wrappers when COLEARN_HOST_SHIM is defined (inside namespace colearn).
#pragma once

#ifndef __grid_constant__
#define __grid_constant__
#endif

// ---- shared-window addresses ---------------------------------------------------------------------------------------
// smem_u32(p) = byte offset of p from the 1024-aligned base of the CTA's dynamic shared memory (+ 1024, so that 0 is
// never a valid address).  The swizzle is a function of these address bits, as on the device.
inline uint8_t* shim_smem_base() {
  uintptr_t p = reinterpret_cast<uintptr_t>(::colearn_shim::dyn_smem());
  return reinterpret_cast<uint8_t*>((p + 1023) & ~(uintptr_t)1023);
}
inline uint32_t smem_u32(const void* p) { return (uint32_t)(reinterpret_cast<const uint8_t*>(p) - shim_smem_base()) + 1024u; }
inline uint8_t* shim_smem_ptr(uint32_t saddr) { return shim_smem_base() + (saddr - 1024u); }

// ---- mbarrier ------------------------------------------------------------------------------------------------------
// one 64-bit word: [0] phase parity | [1,17) pending arrivals | [17,33) arrivals per phase | [33,64) pending tx bytes (signed)
struct ShimMbar {
  static uint64_t pack(uint64_t phase, uint64_t pending, uint64_t init, int64_t tx) {
    return (phase & 1) | ((pending & 0xFFFF) << 1) | ((init & 0xFFFF) << 17) | ((uint64_t)(tx & 0x7FFFFFFF) << 33);
  }
  static void unpack(uint64_t w, uint64_t& phase, uint64_t& pending, uint64_t& init, int64_t& tx) {
    phase = w & 1;
    pending = (w >> 1) & 0xFFFF;
    init = (w >> 17) & 0xFFFF;
    tx = (int64_t)((w >> 33) & 0x7FFFFFFF);
    if (tx & 0x40000000) tx -= 0x80000000ll;     // sign-extend 31 bits
  }
  // arrivals -= d_arrive, tx += d_tx; the phase completes (flips, arrivals re-armed) when both reach zero
  static void update(uint64_t* bar, int d_arrive, int64_t d_tx) {
    uint64_t old = __atomic_load_n(bar, __ATOMIC_ACQUIRE), want;
    do {
      uint64_t phase, pending, init;
      int64_t tx;
      unpack(old, phase, pending, init, tx);
      if ((int)pending < d_arrive) abort();      // more arrivals than the barrier was initialised for: a protocol bug
      pending -= (uint64_t)d_arrive;
      tx += d_tx;
      if (pending == 0 && tx == 0) {
        phase ^= 1;
        pending = init;
      }
      want = pack(phase, pending, init, tx);
    } while (!__atomic_compare_exchange_n(bar, &old, want, false, __ATOMIC_ACQ_REL, __ATOMIC_ACQUIRE));
  }
};
inline void mbar_init(uint64_t* bar, uint32_t count) { __atomic_store_n(bar, ShimMbar::pack(0, count, count, 0), __ATOMIC_RELEASE); }
inline void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) { ShimMbar::update(bar, 1, (int64_t)bytes); }
inline void mbar_arrive(uint64_t* bar) { ShimMbar::update(bar, 1, 0); }
inline uint32_t mbar_try_wait(uint32_t bar_addr, uint32_t parity) {
  const uint64_t w = __atomic_load_n(reinterpret_cast<uint64_t*>(shim_smem_ptr(bar_addr)), __ATOMIC_ACQUIRE);
  return ((w & 1) != (parity & 1)) ? 1u : 0u;    // the phase with this parity has completed
}
constexpr unsigned long long kMbarTimeoutNs = 20ull * 1000 * 1000 * 1000;
inline void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  const auto t0 = std::chrono::steady_clock::now();
  while (!mbar_try_wait(addr, parity)) {
    std::this_thread::yield();
    if (std::chrono::steady_clock::now() - t0 > std::chrono::nanoseconds(kMbarTimeoutNs)) abort();   // the device traps here
  }
}

// ---- tensor maps + TMA -----------------------------------------------------------------------------------------------
// What cuTensorMapEncodeTiled would encode, kept in the opaque 128 bytes of a CUtensorMap (bf16, SWIZZLE_128B, zero fill)
struct ShimTensorMap {
  const __nv_bfloat16* ptr;
  int rank;
  long long dims[4];            // elements, innermost first
  long long strides[4];         // bytes; strides[0] = 2
  int box[4];
};
static_assert(sizeof(ShimTensorMap) <= sizeof(CUtensorMap), "mock tensor map must fit the opaque descriptor");
inline void shim_encode_tiled(CUtensorMap* out, const void* ptr, int rank, const long long* dims, const long long* strides_bytes, const int* box) {
  ShimTensorMap m;
  memset(&m, 0, sizeof(m));
  m.ptr = static_cast<const __nv_bfloat16*>(ptr);
  m.rank = rank;
  for (int i = 0; i < rank; ++i) {
    m.dims[i] = dims[i];
    m.strides[i] = i == 0 ? 2 : strides_bytes[i - 1];
    m.box[i] = box[i];
  }
  if (box[0] != 64) abort();    // SWIZZLE_128B: one box line = 64 bf16
  memset(out, 0, sizeof(*out));
  memcpy(out, &m, sizeof(m));
}
// box lines (all outer coordinates flattened, innermost outer dim fastest) land as 128-byte lines; line r, 16-byte chunk c
// is stored at chunk position c ^ (r % 8) (the address bits [4,7) ^ [7,10) of a 1024-aligned destination)
inline void shim_tma_load(void* smem_dst, const CUtensorMap* tmap, const int* coord, uint64_t* bar) {
  ShimTensorMap m;
  memcpy(&m, tmap, sizeof(m));
  uint8_t* dst = static_cast<uint8_t*>(smem_dst);
  const uint32_t dst_addr = smem_u32(dst);
  if ((dst_addr - 1024u) % 1024u) abort();       // swizzle atoms need 1024-byte aligned boxes
  long long lines = 1;
  for (int i = 1; i < m.rank; ++i) lines *= m.box[i];
  for (long long r = 0; r < lines; ++r) {
    long long rem = r, off_bytes = 0;
    bool inside = true;
    for (int i = 1; i < m.rank; ++i) {
      const long long idx = coord[i] + rem % m.box[i];
      rem /= m.box[i];
      if (idx < 0 || idx >= m.dims[i]) inside = false;
      off_bytes += idx * m.strides[i];
    }
    for (int c = 0; c < 64; ++c) {
      const long long ci = (long long)coord[0] + c;
      __nv_bfloat16 v = __float2bfloat16(0.f);
      if (inside && ci >= 0 && ci < m.dims[0]) v = *reinterpret_cast<const __nv_bfloat16*>(reinterpret_cast<const uint8_t*>(m.ptr) + off_bytes + ci * 2);
      const uint32_t lin = (uint32_t)r * 128u + (uint32_t)c * 2u;
      const uint32_t addr = dst_addr - 1024u + lin;
      const uint32_t sw = addr ^ (((addr >> 7) & 7u) << 4);
      *reinterpret_cast<__nv_bfloat16*>(shim_smem_base() + sw) = v;
    }
  }
  ShimMbar::update(bar, 0, -(long long)lines * 128);
}
inline void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, int c0, int c1, uint64_t* bar) {
  const int coord[2] = {c0, c1};
  shim_tma_load(smem_dst, tmap, coord, bar);
}
inline void tma_load_4d(void* smem_dst, const CUtensorMap* tmap, int c0, int c1, int c2, int c3, uint64_t* bar) {
  const int coord[4] = {c0, c1, c2, c3};
  shim_tma_load(smem_dst, tmap, coord, bar);
}
inline void tmap_prefetch(const CUtensorMap*) {}
inline void fence_mbarrier_init() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
inline void fence_proxy_async() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }

// ---- wgmma ------------------------------------------------------------------------------------------------------------
inline void wgmma_fence() {}
inline void wgmma_commit() {}
// the model's wgmma runs per thread at issue; completion, as seen by any thread of the warpgroup, means that all 128
// threads have run theirs (the stage they read may be released after this)
template <int N>
inline void wgmma_wait() { ::colearn_shim::named_barrier(8 + (int)(::colearn_shim::t_linear / 128), 128); }
template <int R>
inline void acc_fence(float (&)[R]) {}
template <int N>
inline void set_max_regs() {}
inline void wg_bar_sync(int id) { ::colearn_shim::named_barrier(id, 128); }

inline float shim_ld_bf16(uint32_t addr) {   // addr: un-swizzled byte offset in the shared window
  const uint32_t sw = addr ^ (((addr >> 7) & 7u) << 4);
  return __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(shim_smem_base() + sw));
}
// element (r, k) of a [rows x 16] operand addressed through its sm_90 GMMA descriptor
inline float shim_operand(uint64_t d, bool mn_major, int r, int k) {
  auto field = [](uint64_t x, int lo, int bits) { return (uint32_t)((x >> lo) & ((1ull << bits) - 1)); };
  if (field(d, 62, 2) != 1 || field(d, 49, 3) != 0) abort();                      // SWIZZLE_128B, base offset 0
  const uint32_t start = (field(d, 0, 14) << 4) - 1024u, lbo = field(d, 16, 14) << 4, sbo = field(d, 32, 14) << 4;
  uint32_t addr;
  if (mn_major)   // ((8,n),(8,k)):((1,LBO),(8,SBO)) in 16-byte units: 64 MN elements per line, 8 k-lines per atom
    addr = start + (uint32_t)(r % 64) * 2u + (uint32_t)(r / 64) * lbo + (uint32_t)(k % 8) * 128u + (uint32_t)(k / 8) * sbo;
  else            // K-major: row r = 128-byte line, 8-row groups SBO apart; the start address carries the k offset
    addr = start + (uint32_t)(r % 8) * 128u + (uint32_t)(r / 8) * sbo + (uint32_t)k * 2u;
  return shim_ld_bf16(addr);
}
// one wgmma.mma_async.m64nNk16.f32.bf16.bf16 with scale-d = 1: this thread's share of D[64, N] += A[64, 16] . B[N, 16]^T.
// Fragment: thread t of the warpgroup holds d[4 i + j] = D[16 (t / 32) + (t % 32) / 4 + 8 (j / 2), 8 i + 2 (t % 4) + j % 2].
template <int TA, int TB, int R>
inline void wgmma_bf16(float (&d)[R], uint64_t da, uint64_t db) {
  const int t = (int)(::colearn_shim::t_linear % 128), w = t / 32, l = t % 32;
  float a[2][16];
  for (int h = 0; h < 2; ++h)
    for (int k = 0; k < 16; ++k) a[h][k] = shim_operand(da, TA != 0, 16 * w + l / 4 + 8 * h, k);
  for (int i = 0; i < R / 4; ++i)
    for (int c = 0; c < 2; ++c) {
      float b[16];
      for (int k = 0; k < 16; ++k) b[k] = shim_operand(db, TB != 0, 8 * i + 2 * (l % 4) + c, k);
      for (int h = 0; h < 2; ++h) {
        float acc = d[4 * i + 2 * h + c];
        for (int k = 0; k < 16; ++k) acc += a[h][k] * b[k];
        d[4 * i + 2 * h + c] = acc;
      }
    }
}
inline uint32_t ld_acquire_sys(const uint32_t* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
inline void ready_wait_ge(const uint32_t* p, uint32_t want) { spin_wait_ge(p, want, 64, "ready flag"); }

// ---- cluster forms: not modelled (the tests drive the 1-CTA kernels) -----------------------------------------------------
inline uint32_t cluster_ctarank() { return 0u; }
inline void cluster_sync_all() {}
inline void tma_load_2d_mcast(void*, const CUtensorMap*, int, int, uint64_t*, uint16_t) { abort(); }
inline void mbar_arrive_cluster(uint64_t* bar, uint32_t cta_rank) {
  if (cta_rank != 0) abort();
  ShimMbar::update(bar, 1, 0);
}
