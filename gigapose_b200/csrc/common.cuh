// Shared device-side helpers for the sm_90a kernels: mbarrier / TMA / wgmma descriptor inline PTX.
// Everything here is hand-written PTX for Hopper (compile with -gencode arch=compute_90a,code=sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdint.h>
#include <cstdio>

namespace gp {

// ----------------------------------------------------------------------------------------------------------
// small utilities
// ----------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
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
      "selp.b32 %0, 1, 0, P;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a protocol bug turns into a trap (reported as a CUDA error) instead of a hung GPU.  No printf here: a
// call inside a wgmma pipeline makes ptxas serialise the warpgroup's MMAs.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}

// ----------------------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) -- 2-D tiled loads, completion on an mbarrier
// ----------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// 4-D tile (implicit-GEMM convolution: {channel, x, y, image} of an NHWC plane; out-of-range x / y are zero-filled)
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0, int32_t c1,
                                            int32_t c2, int32_t c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// L2 cache-policy variants (createpolicy-encoded constants as used by CUTLASS' TMA::CacheHintSm90)
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;
__device__ __forceinline__ void tma_load_2d_hint(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0,
                                                 int32_t c1, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
      : "memory");
}

// ----------------------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptors (sm_90a)
// ----------------------------------------------------------------------------------------------------------
// K-major operand tile whose rows are `kRowBytes` wide (== the TMA swizzle span): rows stored densely, groups of 8 rows
// form one swizzle atom.  start address / LBO / SBO in 16-byte units; layout type (bits 62-63): 1=SW128, 2=SW64, 3=SW32.
// A K step of 16 elements inside the atom advances the start address by 32 bytes.
template <int kRowBytes>
__device__ __forceinline__ uint64_t wgmma_desc_kmajor(uint32_t smem_addr) {
  static_assert(kRowBytes == 128 || kRowBytes == 64 || kRowBytes == 32, "swizzle span");
  constexpr uint64_t layout = kRowBytes == 128 ? 1 : (kRowBytes == 64 ? 2 : 3);
  constexpr uint64_t sbo = (8 * kRowBytes) >> 4;       // stride between 8-row groups
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= 1ull << 16;                                     // LBO: ignored for swizzled K-major operands
  d |= sbo << 32;
  d |= layout << 62;
  return d;
}

// MN-major operand (rows = K index, 64 contiguous MN elements = one 128-byte SWIZZLE_128B row per K index, i.e. a
// [K][64] row-major bf16 tile as TMA delivers it): groups of 8 K-rows are SBO = 1024 B apart; LBO (stride between
// 64-element MN blocks) is unused for N = 64.
__device__ __forceinline__ uint64_t wgmma_desc_mnmajor_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= 1ull << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= 1ull << 62;                                     // SWIZZLE_128B
  return d;
}

// Programmatic dependent launch: a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may become
// resident while its predecessor in the stream is still running (its CTAs take SMs as the predecessor's CTAs retire and
// run their prologue: barrier init, descriptor prefetch).  `pdl_wait` blocks until the predecessor grid
// has completed and its writes are visible -- it must precede the first access to anything an earlier kernel wrote (and
// the first write to anything an earlier kernel reads); it is a no-op for a normally launched kernel.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ void named_barrier_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Warpgroup register reallocation (executed by all 128 threads of a warpgroup): a producer warpgroup that only issues
// TMA gives registers back so that the MMA warpgroups can hold their accumulators and the epilogue without spilling.
template <uint32_t kRegs>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <uint32_t kRegs>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }

}  // namespace gp
