// Hopper (sm_90a) primitives used by the implicit-GEMM convolution:
// mbarrier, TMA (cp.async.bulk.tensor), cp.async, wgmma (warpgroup MMA from shared memory, fp32 accumulators in
// registers) and the wgmma shared-memory descriptor.  Inline PTX only.
#pragma once
#include <cuda.h>
#include <stdint.h>

namespace dirb200 {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (kernel error) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  unsigned long long t0;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  while (!mbar_try_wait(bar, parity)) {
    unsigned long long t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    if (t1 - t0 > 4000000000ull) __trap();   // 4 s
  }
}

// One lane of the (fully converged) warp: the single-thread issue of TMA instructions.  Issuing from
// `if (elect_one())` in a CONVERGED warp -- rather than from a divergent `if (lane == 0)` region -- lets the compiler
// keep descriptors / coordinates in uniform registers.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "elect.sync _|P, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- cp.async
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// arrive on `bar` once every cp.async previously issued by this thread has completed (does not raise the
// barrier's pending count: the thread's arrival is part of the barrier's expected count)
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
// generic-proxy smem writes (cp.async, st.shared) -> visible to the async proxy (wgmma operand reads / TMA)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// --------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tmap, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}

// im2col-mode TMA load of an NHWC tensor (rank 4: C, W, H, N): `pixelsPerColumn` output positions starting at the
// base pixel (w, h, n) -- walking the descriptor's bounding box with its traversal strides -- each displaced by the
// filter-tap offset (off_w, off_h); `channelsPerPixel` channels from c; out-of-image elements arrive as zeros.
__device__ __forceinline__ void tma_load_im2col_4d(uint32_t dst, const CUtensorMap* tmap, uint32_t bar, int c, int w,
                                                   int h, int n, uint16_t off_w, uint16_t off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h)
      : "memory");
}

// ------------------------------------------------------------------- wgmma
// A warpgroup (4 consecutive warps, the first one a multiple of 4) computes D[64 x N] (+)= A[64 x 16] * B[16 x N]
// with both operands in shared memory.  Accumulator fragment of thread t (warp w = (t / 32) % 4, lane l = t % 32):
// d[4j + e] (e = 0, 1) is row 16w + l/4, column 8j + 2(l%4) + e; d[4j + 2 + e] the same columns of row 16w + l/4 + 8.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// TA / TB: 0 = the operand is K-major, 1 = MN-major (transposed); accumulate = 0 overwrites D.
#define DIRB_F4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define DIRB_F16(i) DIRB_F4(i), DIRB_F4(i + 4), DIRB_F4(i + 8), DIRB_F4(i + 12)
#define DIRB_R8(a, b, c, e, f, g, h, k) "%" #a ", %" #b ", %" #c ", %" #e ", %" #f ", %" #g ", %" #h ", %" #k ", "
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
      DIRB_R8(0, 1, 2, 3, 4, 5, 6, 7) DIRB_R8(8, 9, 10, 11, 12, 13, 14, 15) DIRB_R8(16, 17, 18, 19, 20, 21, 22, 23)
      "%24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
      : DIRB_F16(0), DIRB_F16(16)
      : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
      DIRB_R8(0, 1, 2, 3, 4, 5, 6, 7) DIRB_R8(8, 9, 10, 11, 12, 13, 14, 15) DIRB_R8(16, 17, 18, 19, 20, 21, 22, 23)
      DIRB_R8(24, 25, 26, 27, 28, 29, 30, 31) DIRB_R8(32, 33, 34, 35, 36, 37, 38, 39) DIRB_R8(40, 41, 42, 43, 44, 45, 46, 47)
      DIRB_R8(48, 49, 50, 51, 52, 53, 54, 55)
      "%56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n}\n"
      : DIRB_F16(0), DIRB_F16(16), DIRB_F16(32), DIRB_F16(48)
      : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}
#undef DIRB_R8
#undef DIRB_F16
#undef DIRB_F4
// D (+)= A * B for a 64 x BN warpgroup tile, BN = 64 or 128
template <int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if constexpr (BN == 128) wgmma_m64n128<TA, TB>(d, adesc, bdesc, accumulate);
  else wgmma_m64n64<TA, TB>(d, adesc, bdesc, accumulate);
}

// ------------------------------------------------------------- descriptors
// wgmma shared-memory matrix descriptor, 128-byte swizzle (layout type 1, bits [62,64)):
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4   bits [49,52) base offset = 0 (tiles start 1024-byte aligned)
// K-major tile  [rows][64 bf16]: rows 128 B apart, 8-row atoms 1024 B apart  -> SBO = 1024, LBO unused.
// MN-major tile [chunk][k rows][64 bf16 of M/N]: k rows 128 B apart, 8-k atoms 1024 B apart (SBO),
//               64-wide M/N chunks `lbo_bytes` apart (LBO).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

}  // namespace tc
}  // namespace dirb200
