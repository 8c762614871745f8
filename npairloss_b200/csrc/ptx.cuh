// ptx.cuh -- thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA).
// Hand-written for this project; bit layouts follow the PTX ISA 8.x wgmma chapter.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace npair {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking test (try_wait may suspend the thread for a system-dependent time)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// 3-D tiled load global -> smem, completion on an mbarrier (complete_tx::bytes)
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* tmap, uint64_t* bar, int32_t c0, int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const void* tmap, uint64_t* bar, int32_t c0, int32_t c1, int32_t c2, int32_t c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// 2-D tiled store smem -> global (bulk async-group completion)
__device__ __forceinline__ void tma_store_2d(const void* tmap, const void* smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------- wgmma (warpgroup MMA)
// Every wgmma of a warpgroup is issued by all 128 threads; the fp32 accumulator lives in their registers (m64nNk16 layout:
// d[4j + {0,1}] = (row 16 * (warp % 4) + lane / 4, columns 8j + 2 * (lane % 4) + {0,1}), d[4j + {2,3}] = the same at row + 8).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across a wgmma it cannot see into
__device__ __forceinline__ void fence_regs(float (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// the 128 accumulator registers of one m64n256 wgmma: operand list and the matching outputs
#define NPAIR_ACC_REGS "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
#define NPAIR_F4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define NPAIR_F16(i) NPAIR_F4(i), NPAIR_F4(i + 4), NPAIR_F4(i + 8), NPAIR_F4(i + 12)
#define NPAIR_ACC_OUTS(d) NPAIR_F16(0), NPAIR_F16(16), NPAIR_F16(32), NPAIR_F16(48), NPAIR_F16(64), NPAIR_F16(80), NPAIR_F16(96), NPAIR_F16(112)
#define NPAIR_WGMMA(TY, A_AND_B, TAIL, ...)                                                       \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" TAIL ", 0;\n\t"                              \
               "wgmma.mma_async.sync.aligned.m64n256k16.f32." TY "." TY " " NPAIR_ACC_REGS ", " A_AND_B ";\n\t}\n" \
               : NPAIR_ACC_OUTS(d) : __VA_ARGS__)

// D[64 x 256] (+)= A[smem desc, 64 x 16] * B[smem desc, 256 x 16]^T, both operands K-major; accumulate iff scale_d != 0
template <bool BF16>
__device__ __forceinline__ void wgmma_m64n256k16_ss(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  if (BF16) NPAIR_WGMMA("bf16", "%128, %129, p, 1, 1, 0, 0", "130", "l"(a_desc), "l"(b_desc), "r"(scale_d));
  else NPAIR_WGMMA("f16", "%128, %129, p, 1, 1, 0, 0", "130", "l"(a_desc), "l"(b_desc), "r"(scale_d));
}
// same with the A operand in registers (m64k16 fragment: a[0] = (r, 2c..2c+1), a[1] = (r+8, ..), a[2] = (r, 2c+8..), a[3] = (r+8, 2c+8..),
// r = 16 * (warp % 4) + lane / 4, c = lane % 4; low half = lower k)
template <bool BF16>
__device__ __forceinline__ void wgmma_m64n256k16_rs(float (&d)[128], const uint32_t (&a)[4], uint64_t b_desc, uint32_t scale_d) {
  if (BF16) NPAIR_WGMMA("bf16", "{%128, %129, %130, %131}, %132, p, 1, 1, 0", "133", "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(scale_d));
  else NPAIR_WGMMA("f16", "{%128, %129, %130, %131}, %132, p, 1, 1, 0", "133", "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(scale_d));
}
#undef NPAIR_WGMMA
#undef NPAIR_ACC_OUTS
#undef NPAIR_F16
#undef NPAIR_F4
#undef NPAIR_ACC_REGS

// Shared-memory matrix descriptor (sm_90 wgmma) for a K-major operand tile whose rows are exactly one swizzle span wide
// (SWIZZLE_128B: 64 x 2-byte elements per row; SWIZZLE_64B: 32).  8-row groups are `sbo_bytes` apart.
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4 (ignored for swizzled K-major; 1)
//   bits [32,46) stride byte offset >> 4   bits [62,64) layout: 0 none, 1 128B, 2 64B, 3 32B
// Advancing K by 16 elements inside the swizzle span adds 32 bytes to the start address.
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t smem_addr, uint32_t sbo_bytes, uint32_t layout_type) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(layout_type & 3) << 62;
  return d;
}
// K-major, no swizzle (layout type 0): 8 x 16-byte core matrices, lbo = byte distance between the two core matrices of a K=16 step,
// sbo = between 8-row groups
__device__ __forceinline__ uint64_t make_nosw_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}

}  // namespace ptx
}  // namespace npair
