// Shared device-side primitives for the sm_90a kernels: mbarrier, TMA (cp.async.bulk.tensor), the wgmma
// shared-memory matrix descriptor.  Hand-written inline PTX; no CUTLASS/CuTe.  Bit layouts follow the PTX ISA
// "Asynchronous Warpgroup Level Matrix" chapter.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda.h>
#include <stdint.h>

#define VLY_DEVINL __device__ __forceinline__

namespace vly {

// ------------------------------------------------------------------------------------------
// misc
// ------------------------------------------------------------------------------------------
VLY_DEVINL uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

VLY_DEVINL uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
VLY_DEVINL float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
VLY_DEVINL float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
VLY_DEVINL float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// ------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------
VLY_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
VLY_DEVINL void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }

VLY_DEVINL void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
VLY_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
VLY_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
VLY_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ------------------------------------------------------------------------------------------
// TMA
// ------------------------------------------------------------------------------------------
VLY_DEVINL void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2D tile load: c0 = innermost (contiguous) coordinate, c1 = row coordinate.
VLY_DEVINL void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
VLY_DEVINL void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// 1-D bulk copy global -> shared (TMA engine, no tensor map): size multiple of 16 B, both addresses 16 B aligned.
VLY_DEVINL void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// The same copy with an L2 cache-eviction policy (from createpolicy).
VLY_DEVINL void bulk_load_1d_hint(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint64_t policy) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;\n" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
               : "memory");
}
VLY_DEVINL uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;\n" : "=l"(p));
  return p;
}
// Programmatic dependent launch: wait = all memory of the prerequisite grids is visible; launch_dependents = the
// next grid in the stream may start being scheduled (it still blocks in ITS wait until this grid has completed).
VLY_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;\n" ::: "memory"); }
VLY_DEVINL void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory"); }

// ------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor (sm_90a), 128-byte swizzle:
//  start[0,14) LBO[16,30) SBO[32,46) (all in 16-byte units), base_offset[49,52) = 0 (1024-byte aligned atoms),
//  layout[62,64) = 1 (SWIZZLE_128B).
//  K-major operand : rows of 128 B (64 bf16 of K), 8-row atoms of 1024 B;  SBO = 1024 (next 8 rows), LBO unused.
//  MN-major operand: "rows" are K-slices of 128 B (64 bf16 of M/N), 8 of them per 1024 B atom;
//                    SBO = 1024 (next 8 K), LBO = byte distance between 64-element M/N chunks.
// Advancing K by 16 elements inside a K-major atom is +32 B, i.e. +2 in the start field.
// ------------------------------------------------------------------------------------------
VLY_DEVINL uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= uint64_t((smem_addr >> 4) & 0x3FFF);
  d |= uint64_t((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= uint64_t((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= uint64_t(1) << 62;  // SWIZZLE_128B
  return d;
}

VLY_DEVINL float fast_exp2(float x) {  // MUFU.EX2; exp2(-inf) = 0
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

VLY_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
VLY_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// arg-max over a warp: the largest value, the lowest index among equal values (torch.argmax's rule); every lane ends with it
VLY_DEVINL void warp_argmax(float& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
  }
}

}  // namespace vly
