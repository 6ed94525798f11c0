// match_tc.cu -- wgmma tensor-core matcher with exact FP32 re-score.
//
// Behavioural spec: the results are those of reference FindMaxCorr10 / MatchSiftData
// (matching.cu:301-397, 1090-1206), bit for bit -- see match.cu for the semantics.
// The reference evaluates all N1 x N2 x 128 products on the FP32 SIMT pipe; here the dense
// contraction runs on the Hopper tensor cores and only the handful of candidates
// that can decide a row are re-scored with the reference's sequential FMA chain.
//
// Pipeline (3 launches + the exact fallback for rows that cannot be certified):
//   1. prep      both descriptor sets -> split FP16 (hi + lo of the 2^12-scaled value), written
//                directly in the GMMA "interleaved" (no-swizzle, K-major) core-matrix layout so that an
//                operand tile is one contiguous blob = one cp.async.bulk; row norms for the error bound.
//   2. gemm      persistent warp-specialised kernel: a cp.async.bulk producer warp and two consumer
//                warpgroups (64 rows each) that issue wgmma.mma_async m64n128k16 (F16 in, FP32 accumulators in
//                registers; three MMAs per K step: hi*hi + hi*lo + lo*hi) with both operands in shared memory,
//                and keep, per (row, partition), the three largest 4-candidate group maxima.
//   3. resolve   eight lanes per row: merge the segments, certify, exact k=0..127 FMA chains for the
//                surviving candidates, the reference's per-partition update rule and 8-way merge.
#include "common.cuh"

#include <cuda_fp16.h>

namespace cs {

#define TC_KCH 16           // 16-byte chunks (8 halves) per descriptor

// ------------------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
  uint32_t addr = smem_u32(bar), ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// GMMA shared-memory descriptor, K-major, no swizzle ("interleaved" core matrices of
// 8 rows x 16 bytes).  lbo = byte distance between the two K chunks of one K=16 step,
// sbo = byte distance between consecutive 8-row groups (PTX ISA, "Matrix Descriptor Format").
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo)
{
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((lbo >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3FFF) << 32);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// The accumulators are in/out operands so that no consumer is scheduled above the wait.
__device__ __forceinline__ void wg_wait0(float (&d)[64])
{
#pragma unroll
  for (int i = 0; i < 64; i++) asm volatile("" : "+f"(d[i])::"memory");
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
  for (int i = 0; i < 64; i++) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, F16 operands from shared memory, FP32 accumulators.
// Fragment of thread t of the warpgroup: d[4j + 2r + c] = D[16 (t / 32) + (t % 32) / 4 + 8r][8j + 2 (t % 4) + c].
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, int accumulate)
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
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

// ------------------------------------------------------------------------------ workspace
struct TcPlan {
  int n1, n2v, n_mt, n_nt, total, U, runs, grid;
  // experiments (env CS_TC_DBG, results are wrong when set): 1 = B tiles are not reloaded, 2 = MMAs without
  // the top-3 update.  The bit-2 branch in t3_gemm_kernel also keeps the top-3 update below the consumers' release
  // of the B stage: without it, ptxas moves part of the update above that arrive.  Pin the order explicitly before
  // this field goes.
  int dbg;
};
// slot of (cta, run, row-in-tile)
__device__ __forceinline__ size_t tc_slot(const TcPlan &pl, int cta, int run, int rowInTile)
{
  return ((size_t)cta * pl.runs + run) * 128 + rowInTile;   // 128 = rows per CTA tile (T3_MT)
}

// ------------------------------------------------------------------------------ single-pass matcher
// Split-FP16 operands (K_eff = 384), top-3 tracking, fused resolve.
// Every descriptor x (scaled by 2^12 so that the low parts stay FP16-normal) is split into
// hi = fp16(x) and lo = fp16(x - hi); the tensor cores accumulate hi*hi + hi*lo + lo*hi in FP32
// (three wgmma per K=16 step on the same accumulator), which differs from the reference's
// FP32 chain by at most eps = T3_C1*|a|*max|b| -- 27x tighter than plain FP16.  That makes a
// single GEMM pass sufficient: the epilogue keeps, per (row, partition), the three largest
// 4-candidate group maxima (with the ids of the first two); a partition is certified when the
// third lies more than delta = 2*eps below what can still matter, and then only the groups of the
// first (and, if within delta, the second) maximum are re-scored with the exact FMA chain by the
// resolve kernel, which also applies the reference's update rule and 8-way merge.  The two consumer
// warpgroups share the tensor cores: while one runs its MMAs the other updates its top-3 tables.
#define T3_M 64                     // rows per consumer warpgroup (wgmma M)
#define T3_MT 128                   // rows per CTA tile (two consumer warpgroups)
#define T3_N 128                    // candidates per stage (wgmma N)
#define T3_A_PART (T3_MT * 256)     // 32 KB: hi (or lo) halves of an A tile, [chunk][128 rows][16 B]
#define T3_A_BYTES (2 * T3_A_PART)  // 64 KB
#define T3_B_PART (T3_N * 256)      // 32 KB: [chunk][128 rows][16 B]
#define T3_B_BYTES (2 * T3_B_PART)  // 64 KB
#define T3_STAGES 2                 // B stages (A tile + 2 stages = 192 KB of the 227 KB a CTA can have)
#define T3_THREADS 384              // warp 0: producer; warpgroups 1 and 2: consumers
#define T3_SMEM_BYTES (T3_A_BYTES + T3_STAGES * T3_B_BYTES + 1024)
#define T3_PM 40                    // words per (row, segment): g1[8] g2[8] g3[8] i1[8] i2[8]
#define T3_SCALE 4096.0f            // 2^12 per operand -> scores carry 2^24
#define T3_UNSCALE (1.0f / 16777216.0f)
#define T3_LIMIT 8.0f               // |x| < 8 keeps 2^12*x inside FP16
// dropped lo*lo and residuals 3*2^-22, tensor accumulation 2^-15, reference chain 2^-17
#define T3_C1 4.0e-5f
#define T3_C2 1.0e-9f

struct T3Buffers {
  __half *a16, *b16;          // packed hi/lo operand tiles
  float *normA;               // per row of set 1
  float *bmax;                // [0] max norm of set 2 (float bits), [1] bad-input flag
  float *pm;                  // per (row, segment) top-3 tables
  int *fbRows;                // fallback row list
  unsigned int *counters;     // [0] fallback rows, [1] candidate groups re-scored, [2] chains
};

// block = 32 rows x 16 chunks; one launch converts both sets (CTAs [0, blocksA) take set 1)
__global__ void __launch_bounds__(512)
t3_prep_kernel(const SiftPoint *__restrict__ ptsA, int nA, __half *__restrict__ outA, float *__restrict__ norms,
               int blocksA, const SiftPoint *__restrict__ ptsB, int nB, __half *__restrict__ outB,
               float *__restrict__ bmax, float *__restrict__ nextFlags)
{
  __shared__ float s_sq[16][33];
  __shared__ int s_bad;
  if (blockIdx.x == 0 && threadIdx.x < 16) nextFlags[threadIdx.x] = 0.0f;   // the next call's flag area
  const int isB = (int)blockIdx.x >= blocksA;
  const SiftPoint *__restrict__ pts = isB ? ptsB : ptsA;
  const int nvalid = isB ? nB : nA;
  const int lane = threadIdx.x & 31, c = threadIdx.x >> 5;
  const int row = (isB ? (int)blockIdx.x - blocksA : (int)blockIdx.x) * 32 + lane;
  if (threadIdx.x == 0) s_bad = 0;
  __syncthreads();
  float v[8];
  if (row < nvalid) {
    const float4 *p = reinterpret_cast<const float4 *>(pts[row].data + 8 * c);
    float4 a = __ldg(p), b = __ldg(p + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = 0.0f;
  }
  float sq = 0.0f;
  bool bad = false;
  __half hi[8], lo[8];
#pragma unroll
  for (int i = 0; i < 8; i++) {
    sq = fmaf(v[i], v[i], sq);
    bad = bad || !(fabsf(v[i]) < T3_LIMIT);     // also catches NaN/Inf
    const float x = v[i] * T3_SCALE;            // exact
    hi[i] = __float2half_rn(x);
    lo[i] = __float2half_rn(x - __half2float(hi[i]));   // the difference is exact in FP32
  }
  if (bad) s_bad = 1;
  uint4 ph, pl;
  ph.x = (uint32_t)__half_as_ushort(hi[0]) | ((uint32_t)__half_as_ushort(hi[1]) << 16);
  ph.y = (uint32_t)__half_as_ushort(hi[2]) | ((uint32_t)__half_as_ushort(hi[3]) << 16);
  ph.z = (uint32_t)__half_as_ushort(hi[4]) | ((uint32_t)__half_as_ushort(hi[5]) << 16);
  ph.w = (uint32_t)__half_as_ushort(hi[6]) | ((uint32_t)__half_as_ushort(hi[7]) << 16);
  pl.x = (uint32_t)__half_as_ushort(lo[0]) | ((uint32_t)__half_as_ushort(lo[1]) << 16);
  pl.y = (uint32_t)__half_as_ushort(lo[2]) | ((uint32_t)__half_as_ushort(lo[3]) << 16);
  pl.z = (uint32_t)__half_as_ushort(lo[4]) | ((uint32_t)__half_as_ushort(lo[5]) << 16);
  pl.w = (uint32_t)__half_as_ushort(lo[6]) | ((uint32_t)__half_as_ushort(lo[7]) << 16);
  if (!isB) {
    const int tile = row / T3_MT, r = row - tile * T3_MT;
    uint8_t *base = reinterpret_cast<uint8_t *>(outA) + (size_t)tile * T3_A_BYTES + ((size_t)c * T3_MT + r) * 16;
    *reinterpret_cast<uint4 *>(base) = ph;
    *reinterpret_cast<uint4 *>(base + T3_A_PART) = pl;
  } else {
    const int tile = row / T3_N, r = row - tile * T3_N;
    uint8_t *base = reinterpret_cast<uint8_t *>(outB) + (size_t)tile * T3_B_BYTES + ((size_t)c * T3_N + r) * 16;
    *reinterpret_cast<uint4 *>(base) = ph;
    *reinterpret_cast<uint4 *>(base + T3_B_PART) = pl;
  }
  s_sq[c][lane] = sq;
  __syncthreads();
  if (c == 0) {
    float t = 0.0f;
#pragma unroll
    for (int i = 0; i < 16; i++) t += s_sq[i][lane];
    float nrm = sqrtf(t) * 1.0001f;
    if (!isB && row < nvalid) norms[row] = nrm;
    if (isB) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) nrm = fmaxf(nrm, __shfl_xor_sync(0xffffffffu, nrm, o));
      if (lane == 0) atomicMax(reinterpret_cast<int *>(bmax), __float_as_int(nrm));
    }
    if (lane == 0 && s_bad) atomicMax(reinterpret_cast<int *>(bmax) + 1, 1);
  }
}

__global__ void __launch_bounds__(T3_THREADS, 1)
t3_gemm_kernel(const TcPlan pl, const T3Buffers bf)
{
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t *sA = smem;                  // the A tile of the current run
  uint8_t *sB = smem + T3_A_BYTES;     // T3_STAGES x 64 KB
  __shared__ uint64_t bar_a_full, bar_a_empty, bar_b_full[T3_STAGES], bar_b_empty[T3_STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cta = blockIdx.x;
  const int u_begin = min(cta * pl.U, pl.total), u_end = min(u_begin + pl.U, pl.total);

  if (threadIdx.x == 0) {
    // the empty barriers take one arrival per consumer warp (8): each warp's wgmma.wait_group covers its own reads
    mbar_init(&bar_a_full, 1); mbar_init(&bar_a_empty, 8);
    for (int s = 0; s < T3_STAGES; s++) { mbar_init(&bar_b_full[s], 1); mbar_init(&bar_b_empty[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    // ============================ producer: bulk copies of whole operand tiles ============================
    if (lane == 0) {
      int runIdx = 0, prevMt = -1;
      for (int u = u_begin, i = 0; u < u_end; u++, i++) {
        const int mt = u / pl.n_nt, nt = u - mt * pl.n_nt;
        if (mt != prevMt) {
          // every MMA of the previous run must have read the A tile before it is overwritten
          if (runIdx > 0) mbar_wait(&bar_a_empty, (runIdx - 1) & 1);
          mbar_expect_tx(&bar_a_full, T3_A_BYTES);
          bulk_g2s(sA, reinterpret_cast<const uint8_t *>(bf.a16) + (size_t)mt * T3_A_BYTES, T3_A_BYTES, &bar_a_full);
          prevMt = mt; runIdx++;
        }
        const int s = i % T3_STAGES, it = i / T3_STAGES;
        if (it > 0) mbar_wait(&bar_b_empty[s], (it - 1) & 1);
        if ((pl.dbg & 1) && it > 0) { mbar_arrive(&bar_b_full[s]); continue; }   // experiment: no B traffic
        mbar_expect_tx(&bar_b_full[s], T3_B_BYTES);
        bulk_g2s(sB + s * T3_B_BYTES, reinterpret_cast<const uint8_t *>(bf.b16) + (size_t)nt * T3_B_BYTES, T3_B_BYTES, &bar_b_full[s]);
      }
    }
  } else if (warp >= 4) {
    // ============================ consumers: MMAs and top-3 tables, one warpgroup per 64 rows ============================
    const unsigned int FULL = 0xffffffffu;
    const int g = (warp - 4) >> 2, wi = warp & 3;
    const int hb = (lane >> 1) & 1;       // this lane's 4-candidate groups are those of the partitions of parity hb
    const int rowInTile = g * T3_M + 16 * wi + (lane >> 2);   // and +8 (accumulator fragment rows)
    const uint32_t aBase = smem_u32(sA) + g * T3_M * 16, bBase = smem_u32(sB);
    float acc[64];
#pragma unroll
    for (int e = 0; e < 64; e++) acc[e] = 0.0f;
    // [fragment row][partition 2q + hb]
    float g1[2][4], g2[2][4], g3[2][4];
    int i1[2][4], i2[2][4];
    int prevMt = -1, runIdx = 0;
    size_t slot = 0;
    for (int u = u_begin, i = 0; u < u_end; u++, i++) {
      const int mt = u / pl.n_nt, nt = u - mt * pl.n_nt;
      if (mt != prevMt) {
        slot = tc_slot(pl, cta, runIdx, rowInTile);
        mbar_wait(&bar_a_full, runIdx & 1);
        prevMt = mt; runIdx++;
#pragma unroll
        for (int r = 0; r < 2; r++)
#pragma unroll
          for (int q = 0; q < 4; q++) { g1[r][q] = 0.0f; g2[r][q] = 0.0f; g3[r][q] = 0.0f; i1[r][q] = -1; i2[r][q] = -1; }
      }
      const int s = i % T3_STAGES, it = i / T3_STAGES;
      mbar_wait(&bar_b_full[s], it & 1);
      const uint32_t bS = bBase + s * T3_B_BYTES;
      wg_fence();
#pragma unroll
      for (int k = 0; k < 8; k++) {
        // K=16 step k = chunks 2k, 2k+1 of the [chunk][128 rows][16 B] parts
        const uint64_t ahi = gmma_desc(aBase + 2 * k * (T3_MT * 16), T3_MT * 16, 128);
        const uint64_t alo = gmma_desc(aBase + T3_A_PART + 2 * k * (T3_MT * 16), T3_MT * 16, 128);
        const uint64_t bhi = gmma_desc(bS + 2 * k * (T3_N * 16), T3_N * 16, 128);
        const uint64_t blo = gmma_desc(bS + T3_B_PART + 2 * k * (T3_N * 16), T3_N * 16, 128);
        wgmma_m64n128k16(acc, ahi, bhi, k > 0);
        wgmma_m64n128k16(acc, ahi, blo, 1);
        wgmma_m64n128k16(acc, alo, bhi, 1);
      }
      wg_commit();
      wg_wait0(acc);
      const bool lastOfRun = (u + 1 == u_end) || ((u + 1) / pl.n_nt != mt);
      if (lane == 0) {
        mbar_arrive(&bar_b_empty[s]);
        if (lastOfRun) mbar_arrive(&bar_a_empty);
      }
      if (!(pl.dbg & 2)) {                           // experiment (bit 1): MMAs without the top-3 update
        // columns 8j + 2(lane % 4) + {0, 1}: the lane pair (lane, lane ^ 1) holds group 2j + hb of partition 2(j % 4) + hb
        const int gbase = nt * (T3_N / 4) + hb;
#pragma unroll
        for (int j = 0; j < 16; j++) {
#pragma unroll
          for (int r = 0; r < 2; r++) {
            float v = fmaxf(acc[4 * j + 2 * r], acc[4 * j + 2 * r + 1]);
            v = fmaxf(v, __shfl_xor_sync(FULL, v, 1));
            const int q = j & 3, id = gbase + 2 * j;
            const bool t = v > g1[r][q], u2 = v > g2[r][q];
            g3[r][q] = fmaxf(g3[r][q], fminf(g2[r][q], v));
            i2[r][q] = u2 ? (t ? i1[r][q] : id) : i2[r][q];
            g2[r][q] = fmaxf(g2[r][q], fminf(g1[r][q], v));
            i1[r][q] = t ? id : i1[r][q];
            g1[r][q] = fmaxf(g1[r][q], v);
          }
        }
      }
      if (lastOfRun && !(lane & 1)) {
#pragma unroll
        for (int r = 0; r < 2; r++) {
          float *o = bf.pm + (slot + 8 * r) * T3_PM;
#pragma unroll
          for (int q = 0; q < 4; q++) {
            const int p = 2 * q + hb;
            o[p] = g1[r][q]; o[8 + p] = g2[r][q]; o[16 + p] = g3[r][q];
            o[24 + p] = __int_as_float(i1[r][q]); o[32 + p] = __int_as_float(i2[r][q]);
          }
        }
      }
    }
  }
}

// ---- resolve ---------------------------------------------------------------------------------
// Eight lanes per row (four rows per warp): merge the segments' top-3 tables (lane = partition),
// decide which partitions can matter, re-score their first (and, within delta, second) groups
// exactly (lane = candidate, eight per round), then the reference's per-partition rule
// (matching.cu:354-359, stated order-independently) and 8-way merge (:378-390).
#define T3_RW 4                       // warps per CTA (16 rows)
#define T3_TAB 64                     // exact scores a row can collect (8 partitions x 2 groups x 4)

struct T3ResolveSmem {
  float4 a[T3_RW][4][33];             // the rows' own descriptors (+1: the four rows of a warp hit different banks)
  float sc[T3_RW][4][T3_TAB];         // exact scores
  int p2[T3_RW][4][T3_TAB];           // their indices
  float2 xy[T3_RW][4][T3_TAB];        // their positions (match_xpos / match_ypos)
  int grp[T3_RW][4][16];              // candidate group list
};

__global__ void __launch_bounds__(32 * T3_RW)
t3_resolve_kernel(const TcPlan pl, const T3Buffers bf, SiftPoint *__restrict__ sift1, const SiftPoint *__restrict__ sift2)
{
  __shared__ T3ResolveSmem sm;
  __shared__ unsigned int s_chains;      // one global atomic per CTA: same-address atomics serialise in L2
  if (threadIdx.x == 0) s_chains = 0;
  __syncthreads();
  const unsigned int FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int sub = lane >> 3, p = lane & 7;                   // row within the warp; partition / candidate slot
  const int row = (blockIdx.x * T3_RW + w) * 4 + sub;
  const bool valid = row < pl.n1;
  const int rrow = valid ? row : pl.n1 - 1;                   // clamped: padding lanes mirror the last row
  const int mt = rrow / T3_MT, rowInTile = rrow - mt * T3_MT;
  // the row's descriptor (each lane four float4), needed by every chain
#pragma unroll
  for (int j = 0; j < 4; j++) sm.a[w][sub][p + 8 * j] = __ldg(reinterpret_cast<const float4 *>(sift1[rrow].data) + p + 8 * j);
  const float bmax = __int_as_float(*reinterpret_cast<const int *>(bf.bmax));
  const float normA = bf.normA[rrow];
  // merged top-3 of partition p.  The segments' tables are fetched together (independent loads, one
  // round trip) and inserted afterwards; T3_SEG bounds the unrolled part, more segments take the loop.
  float G = 0.0f, S = 0.0f, Th = 0.0f;
  int I1 = -1, I2 = -1;
  {
    const int u0 = mt * pl.n_nt, u1 = u0 + pl.n_nt - 1;
    const int c0 = u0 / pl.U, c1 = u1 / pl.U;
    auto insert = [&](float v, int id) {
      const bool t = v > G, u2 = v > S;
      Th = fmaxf(Th, fminf(S, v));
      I2 = u2 ? (t ? I1 : id) : I2;
      S = fmaxf(S, fminf(G, v));
      I1 = t ? id : I1;
      G = fmaxf(G, v);
    };
    constexpr int T3_SEG = 6;
    float v[T3_SEG][3];
    int id[T3_SEG][2];
#pragma unroll
    for (int k = 0; k < T3_SEG; k++) {
      const int c = c0 + k;
      if (c <= c1) {
        const int run = mt - (c * pl.U) / pl.n_nt;
        const float *q = bf.pm + tc_slot(pl, c, run, rowInTile) * T3_PM;
        v[k][0] = q[p]; v[k][1] = q[8 + p]; v[k][2] = q[16 + p];
        id[k][0] = __float_as_int(q[24 + p]); id[k][1] = __float_as_int(q[32 + p]);
      } else {
        v[k][0] = v[k][1] = v[k][2] = 0.0f; id[k][0] = id[k][1] = -1;
      }
    }
#pragma unroll
    for (int k = 0; k < T3_SEG; k++) { insert(v[k][0], id[k][0]); insert(v[k][1], id[k][1]); insert(v[k][2], -1); }
    for (int c = c0 + T3_SEG; c <= c1; c++) {
      const int run = mt - (c * pl.U) / pl.n_nt;
      const float *q = bf.pm + tc_slot(pl, c, run, rowInTile) * T3_PM;
      insert(q[p], __float_as_int(q[24 + p])); insert(q[8 + p], __float_as_int(q[32 + p])); insert(q[16 + p], -1);
    }
    G *= T3_UNSCALE; S *= T3_UNSCALE; Th *= T3_UNSCALE;
  }
  const float delta = 2.0f * (T3_C1 * normA * bmax + T3_C2 * (normA + bmax));
  // L = second largest element of the pool {G[0..7], S[0]} (S[0] bounds partition 0's second best, quirk Q9)
  float m1 = __shfl_sync(FULL, S, 0, 8), m2 = 0.0f;
#pragma unroll
  for (int y = 0; y < 8; y++) {
    const float gy = __shfl_sync(FULL, G, y, 8);
    m2 = fmaxf(m2, fminf(m1, gy));
    m1 = fmaxf(m1, gy);
  }
  const float L = m2;
  const bool rowOk = (L > 2.0f * delta) && (L < 3.0e38f);       // the deciding elements are clearly positive
  const bool rel = rowOk && (G >= L - delta);
  const float low = (p == 0 ? fminf(L, G) : G) - delta;        // partition 0 also supplies its second best
  const bool cert = !rel || Th <= 0.0f || Th < low;
  const bool use1 = rel && I1 >= 0;
  const bool use2 = rel && I2 >= 0 && S >= low;
  const unsigned int certMask = (__ballot_sync(FULL, cert) >> (8 * sub)) & 0xffu;
  const bool ok = valid && rowOk && certMask == 0xffu;
  if (valid && !ok && p == 0) {
    // every row lists itself at most once, so the index stays below n1 when the counter started at zero; the clamp
    // keeps a stale counter (a previous call that failed half-way) from writing past the list
    const unsigned at = atomicAdd(&bf.counters[0], 1u);
    if (at < (unsigned)pl.n_mt * T3_MT) bf.fbRows[at] = row;
  }
  // candidate group list (first groups, then second groups)
  const unsigned int b1 = (__ballot_sync(FULL, ok && use1) >> (8 * sub)) & 0xffu;
  const unsigned int b2 = (__ballot_sync(FULL, ok && use2) >> (8 * sub)) & 0xffu;
  const int n1g = __popc(b1), ncand = 4 * (n1g + __popc(b2));
  if (ok && use1) sm.grp[w][sub][__popc(b1 & ((1u << p) - 1))] = I1;
  if (ok && use2) sm.grp[w][sub][n1g + __popc(b2 & ((1u << p) - 1))] = I2;
  __syncwarp();
  int maxc = ncand;
#pragma unroll
  for (int o = 16; o >= 8; o >>= 1) maxc = max(maxc, __shfl_xor_sync(FULL, maxc, o));
  for (int c0 = 0; c0 < maxc; c0 += 8) {
    const int c = c0 + p;
    if (c < ncand) {
      const int p2 = sm.grp[w][sub][c >> 2] * 4 + (c & 3);
      const float4 *bp = reinterpret_cast<const float4 *>(sift2[p2].data);
      const float2 xy = make_float2(sift2[p2].xpos, sift2[p2].ypos);
      // the reference's score: sequential k = 0..127 FMA chain starting from 0 (matching.cu:338-351).
      // Software pipeline: the next eight float4 of the candidate are in flight while eight are consumed.
      float acc = 0.0f;
      float4 bv[8], bn[8];
#pragma unroll
      for (int j = 0; j < 8; j++) bv[j] = __ldg(bp + j);
#pragma unroll
      for (int blk = 0; blk < 4; blk++) {
        if (blk < 3) {
#pragma unroll
          for (int j = 0; j < 8; j++) bn[j] = __ldg(bp + 8 * (blk + 1) + j);
        }
        float4 av[8];
#pragma unroll
        for (int j = 0; j < 8; j++) av[j] = sm.a[w][sub][8 * blk + j];
#pragma unroll
        for (int j = 0; j < 8; j++) {
          acc = __fmaf_rn(av[j].x, bv[j].x, acc);
          acc = __fmaf_rn(av[j].y, bv[j].y, acc);
          acc = __fmaf_rn(av[j].z, bv[j].z, acc);
          acc = __fmaf_rn(av[j].w, bv[j].w, acc);
        }
#pragma unroll
        for (int j = 0; j < 8; j++) bv[j] = bn[j];
      }
      sm.sc[w][sub][c] = acc;
      sm.p2[w][sub][c] = p2;
      sm.xy[w][sub][c] = xy;
    }
  }
  __syncwarp();
  // per-partition rule: lane p scans its row's table for partition p ((p2 >> 2) & 7)
  float pmx = 0.0f, psec = 0.0f;
  int pidx = -1, pent = -1;
  for (int e = 0; e < maxc; e++) {
    if (e < ncand) {
      const int p2 = sm.p2[w][sub][e];
      const float sc = sm.sc[w][sub][e];
      if (((p2 >> 2) & 7) == p && sc > 0.0f) {       // a non-positive score cannot match (matching.cu:317-321)
        if (sc > pmx) { psec = pmx; pmx = sc; pidx = p2; pent = e; }
        else {
          if (sc == pmx && p2 < pidx) { pidx = p2; pent = e; }
          psec = fmaxf(psec, sc);
        }
      }
    }
  }
  // 8-way merge, matching.cu:378-390
  float mx = __shfl_sync(FULL, pmx, 0, 8), sec = __shfl_sync(FULL, psec, 0, 8);
  int idx = __shfl_sync(FULL, pidx, 0, 8), ent = __shfl_sync(FULL, pent, 0, 8);
#pragma unroll
  for (int y = 0; y < 8; y++) {
    const float my = __shfl_sync(FULL, pmx, y, 8);
    const int iy = __shfl_sync(FULL, pidx, y, 8), ey = __shfl_sync(FULL, pent, y, 8);
    if (idx != iy) {
      if (my > mx) { sec = fmaxf(mx, sec); mx = my; idx = iy; ent = ey; }
      else if (my > sec) sec = my;
    }
  }
  if (ok && p == 0) {
    SiftPoint *o = sift1 + row;
    const float2 xy = ent >= 0 ? sm.xy[w][sub][ent] : make_float2(0.0f, 0.0f);
    o->score = mx;
    o->match = idx;
    o->match_xpos = xy.x;
    o->match_ypos = xy.y;
    o->ambiguity = __fdiv_rn(sec, __fadd_rn(mx, 1e-6f));
    atomicAdd(&s_chains, (unsigned)ncand);
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_chains) { atomicAdd(&bf.counters[1], s_chains >> 2); atomicAdd(&bf.counters[2], s_chains); }
}

// exact SIMT scan of the rows the tensor path could not certify (match.cu)
int match_exact_fallback(SiftPoint *s1, int n1, const SiftPoint *s2, int n2, const int *rows, const unsigned int *nrows,
                         const unsigned int *gate, cudaStream_t st);

// ------------------------------------------------------------------------------ host
static int ensure(void **p, size_t *cap, size_t bytes)
{
  if (*cap >= bytes) return 0;
  if (*p) cudaFree(*p);
  *p = nullptr; *cap = 0;
  CS_CUDA(cudaMalloc(p, bytes));
  *cap = bytes;
  return 0;
}

bool match_tensor_supported()
{
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return false;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  return major == 9;
}

// One workspace per device, used on the caller's stream: like the reference (function-local static caches,
// cudaSiftH.cu:310,409) the matcher is single-threaded per device -- two host threads matching on the same device at
// the same time would share the tables and the flag areas.
struct T3Workspace {
  T3Buffers bf = {};
  size_t cap[8] = {};
  unsigned int *h_counters = nullptr;
  float *flags = nullptr;         // 2 x 16 words: [0] max norm of set 2, [1] bad-input flag, [4..7] counters
  unsigned long long calls = 0;
  bool dirty = false;             // a call returned with an error after it had started to use the current flag area
  bool configured = false;
  bool pendingStats = false;
};
static T3Workspace g_ws3[16];

// stats: [0] candidate groups re-scored, [1] exact chains, [2] rows that fell back to the exact scan
int match_tensor(SiftPoint *s1, int n1, const SiftPoint *s2, int n2, cudaStream_t st, unsigned long long stats[4])
{
  stats[0] = stats[1] = stats[2] = 0;
  const int n2v = (n2 / 32) * 32;                      // matching.cu:325 (quirk Q7)
  if (n1 <= 0) return 0;
  if (n2v == 0 || !match_tensor_supported()) return match_exact(s1, n1, s2, n2, st);
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  T3Workspace &ws = g_ws3[dev & 15];
  TcPlan pl;
  pl.n1 = n1; pl.n2v = n2v;
  pl.n_mt = idivup(n1, T3_MT); pl.n_nt = idivup(n2v, T3_N);
  pl.total = pl.n_mt * pl.n_nt;
  pl.grid = pl.total < sms ? pl.total : sms;
  pl.U = idivup(pl.total, pl.grid);
  pl.grid = idivup(pl.total, pl.U);
  pl.runs = idivup(pl.U, pl.n_nt) + 1;
  { const char *e = getenv("CS_TC_DBG"); pl.dbg = e ? atoi(e) : 0; }    // experiments, results are wrong when set
  const size_t slots = (size_t)pl.grid * pl.runs * T3_MT;
  const size_t rowsPad = (size_t)pl.n_mt * T3_MT;
  T3Buffers &bf = ws.bf;
  int r;
  if ((r = ensure((void **)&bf.a16, &ws.cap[0], (size_t)pl.n_mt * T3_A_BYTES)) < 0) return r;
  if ((r = ensure((void **)&bf.b16, &ws.cap[1], (size_t)pl.n_nt * T3_B_BYTES)) < 0) return r;
  if ((r = ensure((void **)&bf.normA, &ws.cap[2], rowsPad * sizeof(float))) < 0) return r;
  if ((r = ensure((void **)&bf.pm, &ws.cap[3], slots * T3_PM * sizeof(float))) < 0) return r;
  if ((r = ensure((void **)&bf.fbRows, &ws.cap[4], rowsPad * sizeof(int))) < 0) return r;
  // flags/counters: two 64-byte areas used alternately; a call's prep kernel clears the other one for the
  // next call, which saves a memset node per call
  if (!ws.flags) {
    size_t dummy = 0;
    if ((r = ensure((void **)&ws.flags, &dummy, 128)) < 0) return r;
    CS_CUDA(cudaMemsetAsync(ws.flags, 0, 128, st));
    CS_CUDA(cudaMallocHost((void **)&ws.h_counters, 64));
  }
  bf.bmax = ws.flags + 16 * (ws.calls & 1);
  float *nextFlags = ws.flags + 16 * ((ws.calls + 1) & 1);
  if (ws.dirty) CS_CUDA(cudaMemsetAsync(ws.flags, 0, 128, st));     // a previous call failed between its launches
  ws.dirty = true;                                                  // until this call's launches are all in
  bf.counters = reinterpret_cast<unsigned int *>(bf.bmax) + 4;
  if (!ws.configured) {
    CS_CUDA(cudaFuncSetAttribute(t3_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, T3_SMEM_BYTES));
    ws.configured = true;
  }
  // CUDASIFT_MATCH_TIMING=1: CUDA events between the kernels, printed to stderr (warm caches, unlike ncu)
  static int timing = -1;
  static cudaEvent_t tev[6];
  if (timing < 0) {
    const char *e = getenv("CUDASIFT_MATCH_TIMING");
    timing = (e && atoi(e)) ? 1 : 0;
    if (timing) for (int i = 0; i < 6; i++) cudaEventCreate(&tev[i]);
  }
  if (timing) cudaEventRecord(tev[0], st);
  const int blocksA = pl.n_mt * (T3_MT / 32), blocksB = pl.n_nt * (T3_N / 32);
  if (timing) cudaEventRecord(tev[1], st);
  t3_prep_kernel<<<blocksA + blocksB, 512, 0, st>>>(s1, n1, bf.a16, bf.normA, blocksA, s2, n2v, bf.b16, bf.bmax, nextFlags);
  if (timing) cudaEventRecord(tev[2], st);
  t3_gemm_kernel<<<pl.grid, T3_THREADS, T3_SMEM_BYTES, st>>>(pl, bf);
  if (timing) cudaEventRecord(tev[3], st);
  t3_resolve_kernel<<<idivup(n1, 4 * T3_RW), 32 * T3_RW, 0, st>>>(pl, bf, s1, s2);
  if (timing) cudaEventRecord(tev[4], st);
  count_launch(3);
  CS_CUDA(cudaGetLastError());
  // rows that could not be certified -- or, for inputs the split cannot bound (|x| >= 8, NaN, Inf), every row --
  // go through the exact kernel; which of the two is decided on the device
  if ((r = match_exact_fallback(s1, n1, s2, n2, bf.fbRows, bf.counters, reinterpret_cast<const unsigned int *>(bf.bmax) + 1, st)) < 0) return r;
  if (timing) {
    cudaEventRecord(tev[5], st);
    cudaEventSynchronize(tev[5]);
    float ms[5];
    for (int i = 0; i < 5; i++) cudaEventElapsedTime(&ms[i], tev[i], tev[i + 1]);
    fprintf(stderr, "match timing %dx%d [us]: memset %.1f prep %.1f gemm %.1f resolve %.1f exact-fallback %.1f\n", n1, n2,
            ms[0] * 1e3f, ms[1] * 1e3f, ms[2] * 1e3f, ms[3] * 1e3f, ms[4] * 1e3f);
  }
  CS_CUDA(cudaMemcpyAsync(ws.h_counters, bf.bmax, 64, cudaMemcpyDeviceToHost, st));
  ws.calls++;                           // the prep kernel of this call cleared the other flag area for the next one
  ws.dirty = false;
  ws.pendingStats = true;               // read by match_tensor_stats() after the caller's synchronize
  return 0;
}

// statistics of the last match_tensor on this device (call after the stream was synchronized)
void match_tensor_stats(unsigned long long stats[4])
{
  int dev = 0;
  cudaGetDevice(&dev);
  T3Workspace &ws = g_ws3[dev & 15];
  if (!ws.pendingStats) return;
  ws.pendingStats = false;
  if (ws.h_counters[1] != 0) { stats[0] = stats[1] = 0; stats[2] = ~0ull; return; }   // everything went the exact way
  stats[0] = ws.h_counters[4 + 1];
  stats[1] = ws.h_counters[4 + 2];
  stats[2] = ws.h_counters[4 + 0];
}

}  // namespace cs
