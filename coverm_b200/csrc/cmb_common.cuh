// Shared constants and PTX helpers of the libcoverm_b200 kernels (included inside an anonymous namespace).
#pragma once


constexpr uint32_t SPAN = 32;                   // elements per span = one 128-B tile row; contig alignment
constexpr uint32_t K2_THREADS = 256;
constexpr uint32_t CHUNK = SPAN * K2_THREADS;   // 8192 elements = 32 KB
constexpr uint32_t CHUNK_BYTES = CHUNK * 4;
constexpr uint32_t CHUNK_SPANS = K2_THREADS;    // spans per chunk
constexpr uint32_t ROW_ELEMS = SPAN;            // TMA row: 32 x i32 = 128 B
constexpr uint32_t CHUNK_ROWS = CHUNK / ROW_ELEMS;  // 256
#ifndef CMB_K2_STAGES
#define CMB_K2_STAGES 2
#endif
constexpr uint32_t K2_STAGES = CMB_K2_STAGES;
constexpr uint32_t K2_WARPS = K2_THREADS / 32;  // 8 = span-bitmap words per chunk = K2 warps per CTA
// Span occupancy bitmap: one bit per span (K1 sets it for every event it adds), 8 u32 words per chunk.
constexpr uint32_t BITMAP_SPANS_PER_WORD = 32;
constexpr uint32_t BITMAP_ELEMS_PER_WORD = BITMAP_SPANS_PER_WORD * SPAN;  // 1024
#ifndef CMB_K2_MINBLOCKS
#define CMB_K2_MINBLOCKS 3
#endif
constexpr uint32_t K1_THREADS = 256;

// error_flags bits (device)
constexpr uint32_t ERR_UNSORTED = 1u, ERR_NM = 2u, ERR_BOUNDS = 4u, ERR_CAPACITY = 8u, ERR_TID = 16u, ERR_INTERNAL = 32u;

#define FULL 0xffffffffu

// ------------------------------------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
// TMA: 2-D tiled bulk tensor load global -> shared, completion on an mbarrier.
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tmap, int32_t x, int32_t y, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(x), "r"(y), "r"(bar)
      : "memory");
}

// Order this thread's earlier generic-proxy shared-memory accesses (and, after a CTA barrier, every thread's) before a later
// async-proxy (TMA) write to the same bytes.
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// cp.async: 16 B global -> shared, L2 only; completion tracked per thread by commit / wait groups.
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Little-endian loads of BAM fields at any byte offset
__device__ __forceinline__ uint32_t ldu32(const uint8_t* p) {
  const uintptr_t a = (uintptr_t)p;
  const uint32_t* q = (const uint32_t*)(a & ~(uintptr_t)3);
  const uint32_t sh = (uint32_t)(a & 3) * 8;
  const uint32_t lo = q[0];
  if (sh == 0) return lo;
  return __funnelshift_r(lo, q[1], sh);
}
__device__ __forceinline__ uint32_t ldu16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }

__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULL, v, d);
  return v;
}

