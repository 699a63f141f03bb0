// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor) and the wgmma matrix descriptors.
// Hand-written; bit layouts follow the PTX ISA "wgmma matrix descriptor" table.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mdb {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// non-blocking: has the phase with the given parity completed?
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Blocking wait for the phase with the given parity.  MDB_MBAR_WAIT_MODE: 0 = try_wait with a long suspend-time hint
// (the waiting warp may be parked: NANOSLEEP.SYNCS), 1 = try_wait with the default time limit, 2 = test_wait spin.
#ifndef MDB_MBAR_WAIT_MODE
#define MDB_MBAR_WAIT_MODE 0
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
#if MDB_MBAR_WAIT_MODE == 0
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, 0x989680;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
#elif MDB_MBAR_WAIT_MODE == 1
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
#else
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
#endif
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// im2col mode over a (C, W, H, N) map: pixelsPerColumn consecutive output pixels starting at input position (w, h, n),
// each shifted by the filter offset (off_w, off_h); the walk crosses row and image ends, out-of-bounds pixels read as zero.
__device__ __forceinline__ void tma_load_im2col_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c, int w, int h,
                                                   int n, uint16_t off_w, uint16_t off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h)
      : "memory");
}

// ---------------------------------------------------------------- wgmma shared-memory matrix descriptors (sm_90)
//   bits [0,14) start address >> 4   [16,30) leading byte offset >> 4   [32,46) stride byte offset >> 4
//   [49,52) base offset (0: every tile is 1024-byte aligned)   [62,64) layout type: 1 = SWIZZLE_128B
// K-major operand tile whose rows are 128 bytes (64 bf16), written by TMA with CU_TENSOR_MAP_SWIZZLE_128B: 8 rows x 128 B =
// 1024 B between 8-row core-matrix groups (SBO); LBO is unused for a swizzled K-major operand.  Advancing the start address
// by 32 B selects the next 16-wide K slice inside the swizzle atom.
__device__ __forceinline__ uint64_t make_sw128_kmajor_desc(uint32_t smem_addr_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr_bytes >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>((1024u >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// MN-major operand (e.g. a V tile: rows = K, 128 B = 64 N elements per row, 128B swizzle): LBO = bytes between 64-wide
// N atoms, SBO = 1024 B between 8-row K groups.
__device__ __forceinline__ uint64_t make_sw128_mnmajor_desc(uint32_t smem_addr_bytes, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr_bytes >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((1024u >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t pack_f16(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// Activation element type of a kernel instantiation: bf16, or f16 for models whose parameters are fp16.  Accumulation and
// every epilogue stay fp32; only loads, stores and the tensor-core operands change.
template <bool F16>
struct Act {
  using T = __nv_bfloat16;
  using T2 = __nv_bfloat162;
  static __device__ __forceinline__ uint32_t pack(float a, float b) { return pack_bf16(a, b); }
  static __device__ __forceinline__ float2 to_float2(T2 v) { return __bfloat1622float2(v); }
  static __device__ __forceinline__ float to_float(T v) { return __bfloat162float(v); }
  static __device__ __forceinline__ T from_float(float v) { return __float2bfloat16_rn(v); }
};
template <>
struct Act<true> {
  using T = __half;
  using T2 = __half2;
  static __device__ __forceinline__ uint32_t pack(float a, float b) { return pack_f16(a, b); }
  static __device__ __forceinline__ float2 to_float2(T2 v) { return __half22float2(v); }
  static __device__ __forceinline__ float to_float(T v) { return __half2float(v); }
  static __device__ __forceinline__ T from_float(float v) { return __float2half_rn(v); }
};

}  // namespace mdb
