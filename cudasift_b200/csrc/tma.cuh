// tma.cuh -- mbarrier, TMA (cp.async.bulk.tensor) and bulk-copy (cp.async.bulk) helpers shared by the pyramid,
// detector and tensor-core matcher kernels, and the FP32-pair (f32x2) arithmetic of the pyramid and detector (sm_90a).
#pragma once

#include <cuda.h>   // CUtensorMap (type only: the encoder is resolved at run time, see make_tensor_map_2d)
#include <cuda_runtime.h>
#include <cstdint>

namespace cs {

__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbarrier_init(uint64_t *bar, uint32_t count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbarrier_expect_tx(uint64_t *bar, uint32_t bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbarrier_arrive(uint64_t *bar)
{
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void mbarrier_wait(uint64_t *bar, uint32_t parity)
{
  uint32_t ok, addr = smem_addr(bar);
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void mbarrier_init_fence()
{
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// One box of a 2-D tensor (coordinates in elements, x = innermost; out-of-range elements are zero-filled)
// into shared memory; completion is signalled on `bar` as boxBytes of transaction count.
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, int x, int y, uint64_t *bar)
{
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(smem_addr(dst)), "l"((unsigned long long)map), "r"(x), "r"(y), "r"(smem_addr(bar)) : "memory");
}
// `bytes` contiguous bytes from global into shared memory (both 16-byte aligned, bytes a multiple of 16); completion
// is signalled on `bar` as transaction count.
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}
// Tensor maps that live in global memory (written by the host before the launch): make them visible to
// the TMA unit's descriptor cache before first use.
__device__ __forceinline__ void tensormap_acquire(const CUtensorMap *map)
{
  asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" ::"l"((unsigned long long)map) : "memory");
}

// ---- FP32 pairs: two values travel in one 64-bit register pair (lo, hi).  Hopper has no packed FP32
// instructions, so each half is issued as the scalar round-to-nearest operation (explicit __f*_rn: no
// contraction), which is exactly how each half of a packed operation rounds. ----
typedef unsigned long long f32x2;
__device__ __forceinline__ f32x2 pk(float2 v) { f32x2 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(v.x), "f"(v.y)); return r; }
__device__ __forceinline__ f32x2 pk2(float lo, float hi) { f32x2 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ float2 upk(f32x2 v) { float2 r; asm("mov.b64 {%0, %1}, %2;" : "=f"(r.x), "=f"(r.y) : "l"(v)); return r; }
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c)
{
  const float2 x = upk(a), y = upk(b), z = upk(c);
  return pk2(__fmaf_rn(x.x, y.x, z.x), __fmaf_rn(x.y, y.y, z.y));
}
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { const float2 x = upk(a), y = upk(b); return pk2(__fmul_rn(x.x, y.x), __fmul_rn(x.y, y.y)); }
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) { const float2 x = upk(a), y = upk(b); return pk2(__fadd_rn(x.x, y.x), __fadd_rn(x.y, y.y)); }
__device__ __forceinline__ f32x2 sub2(f32x2 a, f32x2 b) { const float2 x = upk(a), y = upk(b); return pk2(__fsub_rn(x.x, y.x), __fsub_rn(x.y, y.y)); }

// ---- host ----
// 2-D float tensor map: dims (w, h), row stride `pitch` floats, box (boxW, boxH), no swizzle, zero fill.
// Returns 0, or a negative CS_E_* code (the image does not meet TMA's alignment rules: base 16-byte
// aligned, pitch a multiple of 4 floats -- callers then take the non-TMA path).
int make_tensor_map_2d(CUtensorMap *out, const float *base, int w, int h, int pitch, int boxW, int boxH);
bool tensor_map_compatible(const float *base, int pitch);

}  // namespace cs
