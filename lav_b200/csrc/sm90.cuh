// Hopper (sm_90a) warpgroup MMA (wgmma) primitives.  Shared-memory operands are K-major SWIZZLE_128B blocks (piece j of
// 128-byte row r stored at piece j ^ (r & 7), 1024-byte aligned), as TMA writes them.
#pragma once
#include <cuda.h>
#include <cudaTypedefs.h>
#include "common.cuh"

namespace lavb {
namespace sm90 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// generic-proxy shared-memory stores -> visible to the async proxy (wgmma operand reads, TMA)
__device__ __forceinline__ void proxy_fence_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier over `threads` threads (id 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// ---- mbarriers and TMA tile loads (cp.async.bulk.tensor completing on an mbarrier's transaction count)
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  } while (!done);
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// one arrival worth `count` arrivals
__device__ __forceinline__ void mbar_arrive(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}

// ---- TMA tile stores (cp.async.bulk.tensor shared -> global, tracked in bulk groups of the issuing thread).  The data must be
// visible to the async proxy first: every writing thread runs proxy_fence_async() before the barrier that precedes the store.
// Box elements outside the tensor are not written.
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's bulk groups still read their shared-memory source (the source may be overwritten after this)
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// at most N of this thread's bulk groups incomplete (their global writes done)
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// host: cuTensorMapEncodeTiled through the runtime's driver entry point (no -lcuda symbol lookup at load time), or null
inline PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }
  return fn;
}

// wgmma shared-memory matrix descriptor of a K-major SWIZZLE_128B operand starting at saddr (1024-byte aligned):
// start >> 4 in [0,14), leading byte offset >> 4 in [16,30) (unused by swizzled K-major layouts: 1), stride byte offset >> 4
// in [32,46) = 1024 B between 8-row groups, layout type in [62,64) = 1 (128-byte swizzle).  Within the 128-byte swizzle atom
// the K16 step k starts 32 k bytes further: descriptor + 2 k.  Rows r0.. of the operand: saddr + 128 r0 (r0 % 8 == 0).
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr) {
  const uint32_t lo = ((saddr & 0x3FFFFu) >> 4) | (1u << 16);
  const uint32_t hi = (1024u >> 4) | (1u << 30);
  return (uint64_t)lo | ((uint64_t)hi << 32);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads/writes across the asynchronous MMAs (fence after wgmma_wait)
template <int N> __device__ __forceinline__ void acc_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T for N = 32, 64, ..., 256: both operands K-major in shared memory, fp32
// accumulators in registers.  Fragment of thread t of the warpgroup: rows 16 (t/32) + (t%32)/4 (+8), columns 8 i + 2 (t%4)
// (+1) for 8-column group i < N/8:
//   d[4i] = (row, col), d[4i+1] = (row, col+1), d[4i+2] = (row+8, col), d[4i+3] = (row+8, col+1).
// So the fragment of one m64nNk16 is the column-wise concatenation of N/32 m64n32k16 fragments: 32-column chunk c is
// d[16c .. 16c+15].  B rows r0.. of a K-major SWIZZLE_128B operand start at descriptor + 8 r0 (128 B rows, r0 % 8 == 0).
template <int N> __device__ void wgmma(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t accumulate);

// operand text of accumulator registers 16c .. 16c + 15 (one 32-column chunk)
#define LAVB_WG_R0 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
#define LAVB_WG_R1 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define LAVB_WG_R2 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
#define LAVB_WG_R3 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define LAVB_WG_R4 "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79"
#define LAVB_WG_R5 "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
#define LAVB_WG_R6 "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111"
#define LAVB_WG_R7 "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
#define LAVB_WG_D4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define LAVB_WG_D16(i) LAVB_WG_D4(i), LAVB_WG_D4(i + 4), LAVB_WG_D4(i + 8), LAVB_WG_D4(i + 12)
// N, the accumulator register list, the operand numbers of a, b and accumulate (N/2, N/2 + 1, N/2 + 2), the "+f" operands
#define LAVB_WGMMA(N, REGS, IA, IB, IP, ...)                                                                         \
  template <> __device__ __forceinline__ void wgmma<N>(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t accumulate) { \
    asm volatile(                                                                                                      \
        "{\n\t.reg .pred p;\n\t"                                                                                       \
        "setp.ne.b32 p, %" #IP ", 0;\n\t"                                                                              \
        "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." LAVB_H16_PTX "." LAVB_H16_PTX " "                            \
        "{" REGS "}, %" #IA ", %" #IB ", p, 1, 1, 0, 0;\n\t}"                                                          \
        : __VA_ARGS__                                                                                                  \
        : "l"(a), "l"(b), "r"(accumulate));                                                                            \
  }
LAVB_WGMMA(32, LAVB_WG_R0, 16, 17, 18, LAVB_WG_D16(0))
LAVB_WGMMA(64, LAVB_WG_R0 ", " LAVB_WG_R1, 32, 33, 34, LAVB_WG_D16(0), LAVB_WG_D16(16))
LAVB_WGMMA(96, LAVB_WG_R0 ", " LAVB_WG_R1 ", " LAVB_WG_R2, 48, 49, 50, LAVB_WG_D16(0), LAVB_WG_D16(16), LAVB_WG_D16(32))
LAVB_WGMMA(128, LAVB_WG_R0 ", " LAVB_WG_R1 ", " LAVB_WG_R2 ", " LAVB_WG_R3, 64, 65, 66,
           LAVB_WG_D16(0), LAVB_WG_D16(16), LAVB_WG_D16(32), LAVB_WG_D16(48))
LAVB_WGMMA(160, LAVB_WG_R0 ", " LAVB_WG_R1 ", " LAVB_WG_R2 ", " LAVB_WG_R3 ", " LAVB_WG_R4, 80, 81, 82,
           LAVB_WG_D16(0), LAVB_WG_D16(16), LAVB_WG_D16(32), LAVB_WG_D16(48), LAVB_WG_D16(64))
LAVB_WGMMA(192, LAVB_WG_R0 ", " LAVB_WG_R1 ", " LAVB_WG_R2 ", " LAVB_WG_R3 ", " LAVB_WG_R4 ", " LAVB_WG_R5, 96, 97, 98,
           LAVB_WG_D16(0), LAVB_WG_D16(16), LAVB_WG_D16(32), LAVB_WG_D16(48), LAVB_WG_D16(64), LAVB_WG_D16(80))
LAVB_WGMMA(224, LAVB_WG_R0 ", " LAVB_WG_R1 ", " LAVB_WG_R2 ", " LAVB_WG_R3 ", " LAVB_WG_R4 ", " LAVB_WG_R5 ", " LAVB_WG_R6,
           112, 113, 114, LAVB_WG_D16(0), LAVB_WG_D16(16), LAVB_WG_D16(32), LAVB_WG_D16(48), LAVB_WG_D16(64), LAVB_WG_D16(80),
           LAVB_WG_D16(96))
LAVB_WGMMA(256, LAVB_WG_R0 ", " LAVB_WG_R1 ", " LAVB_WG_R2 ", " LAVB_WG_R3 ", " LAVB_WG_R4 ", " LAVB_WG_R5 ", " LAVB_WG_R6 ", " LAVB_WG_R7,
           128, 129, 130, LAVB_WG_D16(0), LAVB_WG_D16(16), LAVB_WG_D16(32), LAVB_WG_D16(48), LAVB_WG_D16(64), LAVB_WG_D16(80),
           LAVB_WG_D16(96), LAVB_WG_D16(112))
#undef LAVB_WGMMA
#undef LAVB_WG_D16
#undef LAVB_WG_D4
#undef LAVB_WG_R0
#undef LAVB_WG_R1
#undef LAVB_WG_R2
#undef LAVB_WG_R3
#undef LAVB_WG_R4
#undef LAVB_WG_R5
#undef LAVB_WG_R6
#undef LAVB_WG_R7

}  // namespace sm90
}  // namespace lavb
