// tc_accum_probe.cu -- the tensor matcher's accumulation, measured on its own (test infrastructure only).
//
// One CTA per (A tile, B tile) pair issues the MMA sequence of t3_gemm_kernel (csrc/match_tc.cu): two warpgroups of
// 64 rows, wgmma.mma_async m64n128k16 F16 x F16 -> FP32 with both operands in shared memory in the no-swizzle K-major
// ("interleaved") core-matrix layout, three MMAs per K = 16 step (hi*hi, hi*lo, lo*hi) on one accumulator, eight K
// steps.  The operand tiles arrive already packed ([hi | lo][chunk][128 rows][16 B], 64 KB each) and the raw
// accumulators [128][128] go back, so the caller can compare them with sum hi*hi + hi*lo + lo*hi in float64.
// The probe reads and writes only its own buffers.
#include <cuda_runtime.h>
#include <stdint.h>

#define P_ROWS 128
#define P_PART (P_ROWS * 256)        // 32 KB: hi (or lo) halves of a tile
#define P_TILE (2 * P_PART)          // 64 KB
#define P_SMEM (2 * P_TILE + 1024)

__device__ __forceinline__ uint64_t desc(uint32_t saddr, uint32_t lbo, uint32_t sbo)
{
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((lbo >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3FFF) << 32);
}

__device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, int accumulate)
{
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(accumulate)
      : "memory");
}

__global__ void __launch_bounds__(256, 1) probe_kernel(const uint4 *__restrict__ a, const uint4 *__restrict__ b,
                                                       float *__restrict__ out)
{
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint4 *sA = reinterpret_cast<uint4 *>(smem), *sB = reinterpret_cast<uint4 *>(smem + P_TILE);
  const uint4 *ga = a + (size_t)blockIdx.x * (P_TILE / 16), *gb = b + (size_t)blockIdx.x * (P_TILE / 16);
  for (int i = threadIdx.x; i < P_TILE / 16; i += blockDim.x) { sA[i] = ga[i]; sB[i] = gb[i]; }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy stores -> wgmma operand reads
  __syncthreads();
  const int g = threadIdx.x >> 7, t = threadIdx.x & 127;
  const uint32_t aBase = (uint32_t)__cvta_generic_to_shared(smem) + g * 64 * 16;
  const uint32_t bBase = (uint32_t)__cvta_generic_to_shared(smem + P_TILE);
  float acc[64];
#pragma unroll
  for (int e = 0; e < 64; e++) acc[e] = 0.0f;
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const uint64_t ahi = desc(aBase + 2 * k * (P_ROWS * 16), P_ROWS * 16, 128);
    const uint64_t alo = desc(aBase + P_PART + 2 * k * (P_ROWS * 16), P_ROWS * 16, 128);
    const uint64_t bhi = desc(bBase + 2 * k * (P_ROWS * 16), P_ROWS * 16, 128);
    const uint64_t blo = desc(bBase + P_PART + 2 * k * (P_ROWS * 16), P_ROWS * 16, 128);
    mma(acc, ahi, bhi, k > 0);
    mma(acc, ahi, blo, 1);
    mma(acc, alo, bhi, 1);
  }
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
#pragma unroll
  for (int i = 0; i < 64; i++) asm volatile("" : "+f"(acc[i])::"memory");
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
  for (int i = 0; i < 64; i++) asm volatile("" : "+f"(acc[i])::"memory");
  // d[4j + 2r + c] = D[16 (t / 32) + (t % 32) / 4 + 8r][8j + 2 (t % 4) + c]
  float *o = out + (size_t)blockIdx.x * P_ROWS * P_ROWS;
#pragma unroll
  for (int j = 0; j < 16; j++)
#pragma unroll
    for (int r = 0; r < 2; r++)
#pragma unroll
      for (int c = 0; c < 2; c++)
        o[(size_t)(g * 64 + 16 * (t / 32) + (t % 32) / 4 + 8 * r) * P_ROWS + 8 * j + 2 * (t % 4) + c] = acc[4 * j + 2 * r + c];
}

// a, b: blocks packed tiles each; out: blocks x [128][128] floats.  Returns the CUDA error code (0: success).
extern "C" int probe_run(const void *a, const void *b, float *out, int blocks)
{
  cudaError_t e = cudaFuncSetAttribute(probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, P_SMEM);
  if (e != cudaSuccess) return (int)e;
  probe_kernel<<<blocks, 256, P_SMEM>>>(static_cast<const uint4 *>(a), static_cast<const uint4 *>(b), out);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  return (int)cudaDeviceSynchronize();
}
