// sm_90a primitives used by the tensor-core kernels: mbarrier, TMA (cp.async.bulk[.tensor]), warpgroup MMA
// (wgmma.mma_async with both operands in shared memory, fp32 accumulators in registers) and its shared-memory matrix
// descriptor.  Bit layouts follow the PTX ISA "wgmma matrix descriptor" table (same fields as cute/arch/mma_sm90_desc.hpp).
#pragma once
#include <cstdio>
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace rv {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ----------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// The spin loop lives INSIDE the asm block: a C++ `while (!try_wait)` is a divergent loop to the compiler, after which
// it no longer treats warp-uniform values (descriptors, barrier addresses) as uniform.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "RV_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra RV_DONE;\n\t"
      "bra RV_WAIT;\n\t"
      "RV_DONE:\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

// ---- TMA ---------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* m, uint64_t* bar, void* smem, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// the 3-D box of image c3 of a batched map (4th dimension = image)
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, void* smem, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* smem, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// shared -> global tensor store of one box (out-of-bounds elements are not written), tracked by the issuing thread's
// bulk async-groups: commit after the stores of a buffer, wait_read<0> before that buffer is written again, wait<0> before
// the thread exits
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* smem, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* smem, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* m, const void* smem, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// plain (non-tensor) bulk copy global -> shared; bytes % 16 == 0, both addresses 16-byte aligned
__device__ __forceinline__ void bulk_load(const void* gmem, uint64_t* bar, void* smem, uint32_t bytes) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(gmem)), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// One elected lane of a fully converged warp (TMA issue from warp-uniform control flow).
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
  return pred != 0;
}

// ---- wgmma -------------------------------------------------------------------------------------
// A warpgroup (4 consecutive warps, warp index % 4 == 0 first) issues every wgmma together.  fence: before the first MMA
// that reads / writes accumulator registers the threads touched since; commit + wait<n>: at most n groups still in flight.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// K-major operand tile written by TMA (or the host) with SWIZZLE_128B: rows of 128 bytes (64 x 16-bit), `sbo` bytes
// between 8-row groups.  The start address may be advanced by k*32 bytes to select a 16-element K slice, and by whole
// 128-byte rows: the swizzle is a function of the shared-memory address bits, so such a view reads what TMA wrote.
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr, uint32_t sbo = 1024) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);  // start address      bits [0,14)
  d |= (uint64_t)1 << 16;                    // LBO (unused for swizzled K-major)
  d |= (uint64_t)(sbo >> 4) << 32;           // SBO                bits [32,46)
  d |= (uint64_t)1 << 62;                    // SWIZZLE_128B       bits [62,64) = 1
  return d;
}
// K-major operand tile with SWIZZLE_32B: rows of 32 bytes (16 x 16-bit = one K slice), 8-row groups 256 bytes apart;
// 16-byte chunk j of row r sits at chunk j ^ ((r >> 2) & 1)  (Swizzle<1,4,3>: address bit 4 ^= bit 7).
__device__ __forceinline__ uint64_t desc_sw32(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(256 >> 4) << 32;
  d |= (uint64_t)3 << 62;                    // SWIZZLE_32B
  return d;
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, both K-major in shared memory, fp32 accumulators: thread t of the warpgroup
// holds rows 16 * (t / 32) + (t % 32) / 4 (+ 8) and columns 8 j + 2 (t % 4) (+ 1) as d[4 j + {0, 1}] (+ 8 rows: {2, 3}).
// acc == 0 overwrites D.  One wrapper per N; BF selects bf16 over f16 operands.
#define RV_ACC4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define RV_ACC8(i) RV_ACC4(i), RV_ACC4(i + 4)
#define RV_ACC16(i) RV_ACC8(i), RV_ACC8(i + 8)
// T: operand type, N: columns, REGS: "%0, ..., %(N/2 - 1)", AB: "%(N/2), %(N/2 + 1)", P: "%(N/2 + 2)", then the N/2 accumulators
#define RV_WGMMA(T, N, REGS, AB, P, ...)                                                                      \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " P ", 0;\n\twgmma.mma_async.sync.aligned.m64n" #N "k16.f32." T \
               "." T " {" REGS "}, " AB ", p, 1, 1, 0, 0;\n\t}"                                                \
               : __VA_ARGS__ : "l"(a), "l"(b), "r"(acc))
template <bool BF>
__device__ __forceinline__ void wgmma_m64n16k16(float (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
#define RV_R "%0, %1, %2, %3, %4, %5, %6, %7"
  if constexpr (BF) RV_WGMMA("bf16", 16, RV_R, "%8, %9", "%10", RV_ACC8(0));
  else RV_WGMMA("f16", 16, RV_R, "%8, %9", "%10", RV_ACC8(0));
#undef RV_R
}
template <bool BF>
__device__ __forceinline__ void wgmma_m64n32k16(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
#define RV_R "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
  if constexpr (BF) RV_WGMMA("bf16", 32, RV_R, "%16, %17", "%18", RV_ACC16(0));
  else RV_WGMMA("f16", 32, RV_R, "%16, %17", "%18", RV_ACC16(0));
#undef RV_R
}
template <bool BF>
__device__ __forceinline__ void wgmma_m64n48k16(float (&d)[24], uint64_t a, uint64_t b, uint32_t acc) {
#define RV_R "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23"
  if constexpr (BF) RV_WGMMA("bf16", 48, RV_R, "%24, %25", "%26", RV_ACC16(0), RV_ACC8(16));
  else RV_WGMMA("f16", 48, RV_R, "%24, %25", "%26", RV_ACC16(0), RV_ACC8(16));
#undef RV_R
}
template <bool BF>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
#define RV_R "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
  if constexpr (BF) RV_WGMMA("bf16", 64, RV_R, "%32, %33", "%34", RV_ACC16(0), RV_ACC16(16));
  else RV_WGMMA("f16", 64, RV_R, "%32, %33", "%34", RV_ACC16(0), RV_ACC16(16));
#undef RV_R
}
template <bool BF>
__device__ __forceinline__ void wgmma_m64n80k16(float (&d)[40], uint64_t a, uint64_t b, uint32_t acc) {
#define RV_R "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39"
  if constexpr (BF) RV_WGMMA("bf16", 80, RV_R, "%40, %41", "%42", RV_ACC16(0), RV_ACC16(16), RV_ACC8(32));
  else RV_WGMMA("f16", 80, RV_R, "%40, %41", "%42", RV_ACC16(0), RV_ACC16(16), RV_ACC8(32));
#undef RV_R
}
template <bool BF>
__device__ __forceinline__ void wgmma_m64n96k16(float (&d)[48], uint64_t a, uint64_t b, uint32_t acc) {
#define RV_R "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
  if constexpr (BF) RV_WGMMA("bf16", 96, RV_R, "%48, %49", "%50", RV_ACC16(0), RV_ACC16(16), RV_ACC16(32));
  else RV_WGMMA("f16", 96, RV_R, "%48, %49", "%50", RV_ACC16(0), RV_ACC16(16), RV_ACC16(32));
#undef RV_R
}
template <bool BF>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
#define RV_R "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
  if constexpr (BF) RV_WGMMA("bf16", 128, RV_R, "%64, %65", "%66", RV_ACC16(0), RV_ACC16(16), RV_ACC16(32), RV_ACC16(48));
  else RV_WGMMA("f16", 128, RV_R, "%64, %65", "%66", RV_ACC16(0), RV_ACC16(16), RV_ACC16(32), RV_ACC16(48));
#undef RV_R
}
#undef RV_WGMMA
#undef RV_ACC16
#undef RV_ACC8
#undef RV_ACC4

template <int N, bool BF16>
__device__ __forceinline__ void wgmma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  float (&r)[N / 2] = *reinterpret_cast<float (*)[N / 2]>(d);
#define RV_WG(n) \
  if constexpr (N == n) wgmma_m64n##n##k16<BF16>(r, a, b, acc);
  RV_WG(16) RV_WG(32) RV_WG(48) RV_WG(64) RV_WG(80) RV_WG(96) RV_WG(128)
#undef RV_WG
}

}  // namespace tc

// host: driver entry point for cuTensorMapEncodeTiled without linking libcuda
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                        const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                        const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                        CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_tmapEncodeTiled get_tmap_encoder();

}  // namespace rv
