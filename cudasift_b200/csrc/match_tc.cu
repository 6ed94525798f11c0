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
//                surviving candidates, then the rule: the reference's per-partition update rule and 8-way merge, or
//                the two nearest neighbours.  One kernel, t3_resolve_kernel<KNN, TABLE>, serves both rules.
// Mutual matching uses the same prep launch to convert each set once for both of its roles, runs steps 2 and 3 and
// the exact fallback per direction, then the cross-check (match_mutual.cu).  Two-nearest-neighbour matching
// (match_knn_tensor) runs the same prep and GEMM over all candidates, then the resolve's top-2 rule and the exact top-2
// fallback (match_knn.cu); a batch wave of ratio matching runs them over a table of directions.
#include "common.cuh"
#include "ordered_list.cuh"

#include <cuda_fp16.h>

#include <algorithm>
#include <type_traits>
#include <vector>

namespace cs {

#define TC_KCH 16           // 16-byte chunks (8 halves) per descriptor

// ------------------------------------------------------------------------------ PTX helpers
// (mbarrier and bulk-copy wrappers: tma.cuh)
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
// The GEMM's units (A tile, B tile) are numbered in row-tile order, and CTA c takes units [c U, (c + 1) U).  In a batch
// wave the units of its directions follow each other (MbDir::u0) and U, total and grid cover all of them.
struct TcPlan {
  int n_mt, n_nt, total, U, grid;
};
// The top-3 tables hold one entry per (A tile, segment): the units of row tile t (numbered over all directions of a
// wave) that CTA c runs.  Along the units both t and c only grow and one of them steps at every new segment, so t + c
// numbers the segments without gaps or repeats: slot (t + c) * 128 + row-in-tile, (tiles + grid) * 128 slots.
__device__ __forceinline__ size_t tc_slot(int tile, int cta, int rowInTile)
{
  return (size_t)(tile + cta) * 128 + rowInTile;           // 128 = rows per CTA tile (T3_MT)
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
  float *pm;                  // per (row, segment) top-3 tables
  int *fbRows;                // fallback row list
};

// Chunk c (8 values) of a row's descriptor, zeros for rows >= nvalid: the split halves, the chunk's sum of squares and
// the out-of-range test.
__device__ __forceinline__ void t3_split_chunk(const SiftPoint *__restrict__ pts, int row, int nvalid, int c,
                                               __half (&hi)[8], __half (&lo)[8], float &sq, bool &bad)
{
  float v[8];
  if (row < nvalid) {
    const float4 *p = reinterpret_cast<const float4 *>(pts[row].data + 8 * c);
    float4 a = __ldg(p), b = __ldg(p + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = 0.0f;
  }
  sq = 0.0f;
  bad = false;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    sq = fmaf(v[i], v[i], sq);
    bad = bad || !(fabsf(v[i]) < T3_LIMIT);     // also catches NaN/Inf
    const float x = v[i] * T3_SCALE;            // exact
    hi[i] = __float2half_rn(x);
    lo[i] = __float2half_rn(x - __half2float(hi[i]));   // the difference is exact in FP32
  }
}
// eight halves -> the 16 bytes of one core-matrix row
__device__ __forceinline__ uint4 t3_pack8(const __half (&h)[8])
{
  uint4 p;
  p.x = (uint32_t)__half_as_ushort(h[0]) | ((uint32_t)__half_as_ushort(h[1]) << 16);
  p.y = (uint32_t)__half_as_ushort(h[2]) | ((uint32_t)__half_as_ushort(h[3]) << 16);
  p.z = (uint32_t)__half_as_ushort(h[4]) | ((uint32_t)__half_as_ushort(h[5]) << 16);
  p.w = (uint32_t)__half_as_ushort(h[6]) | ((uint32_t)__half_as_ushort(h[7]) << 16);
  return p;
}

// ---- prep: each set converted once, for both of its roles ---------------------------------------------------------
// In a mutual match a set is the A operand of its own direction (all n rows, with per-row norms) and the B operand of
// the other one (only rows < nv = 32*floor(n/32), quirk Q7, zeros beyond).  The two roles have the same tile layout, so
// `a` serves both unless the tail rows [nv, n) lie in a tile that the B role reads (n % 32 != 0 and nv % 128 != 0);
// then `b` receives a B-role copy of the first bTiles tiles with the tail zeroed.  A one-way match gives set 1 the A
// role only (nv = 0) and set 2 the B role only (n = nv).
static_assert(T3_MT == T3_N && T3_A_PART == T3_B_PART, "A and B operand tiles share one layout");
struct T3PrepSet {
  const SiftPoint *pts;
  int n, nv;
  int blocks;             // CTAs of 32 rows: every A tile of the set
  __half *a, *b;          // b == NULL: `a` is also the B operand
  int bTiles;             // tiles of the B role: ceil(nv / 128)
  float *norms;           // per row, A role
  float *bmax;            // max norm over rows < nv (float bits): the error bound of the other direction
  float *bad;             // batch: the set's bad-input flag
  int blk0;               // batch: its first CTA
};

// block = 32 rows x 16 chunks.  A call: CTAs [0, s0.blocks) take set 1, the rest set 2, a bad value raises *gate.  A
// batch wave (TABLE): the table's sets, each from its blk0 on, each with its own flag.
template <bool TABLE>
__global__ void __launch_bounds__(512)
t3_prep_kernel(const T3PrepSet s0, const T3PrepSet s1, const T3PrepSet *__restrict__ sets, int numSets,
               float *__restrict__ gate, float *__restrict__ nextFlags)
{
  __shared__ float s_sq[16][33];
  __shared__ int s_bad;
  T3PrepSet s;
  int blk;
  if (TABLE) {
    s = sets[table_find(sets, numSets, &T3PrepSet::blk0, (int)blockIdx.x)];
    blk = (int)blockIdx.x - s.blk0;
    gate = s.bad;
  } else {
    if (blockIdx.x == 0 && threadIdx.x < 16) nextFlags[threadIdx.x] = 0.0f;   // the next call's flag area
    const bool second = (int)blockIdx.x >= s0.blocks;
    s = second ? s1 : s0;
    blk = second ? (int)blockIdx.x - s0.blocks : (int)blockIdx.x;
  }
  const int lane = threadIdx.x & 31, c = threadIdx.x >> 5;
  const int row = blk * 32 + lane;
  // nv is a multiple of 32: the CTA's rows lie all below nv (candidates of the other direction) or none of them
  const bool cand = blk * 32 < s.nv;
  if (threadIdx.x == 0) s_bad = 0;
  __syncthreads();
  __half hi[8], lo[8];
  float sq;
  bool bad;
  t3_split_chunk(s.pts, row, s.n, c, hi, lo, sq, bad);
  if (bad) s_bad = 1;
  const uint4 ph = t3_pack8(hi), pl = t3_pack8(lo);
  const int tile = row / T3_MT, r = row - tile * T3_MT;
  const size_t off = (size_t)tile * T3_A_BYTES + ((size_t)c * T3_MT + r) * 16;
  uint8_t *a = reinterpret_cast<uint8_t *>(s.a) + off;
  *reinterpret_cast<uint4 *>(a) = ph;
  *reinterpret_cast<uint4 *>(a + T3_A_PART) = pl;
  if (s.b && tile < s.bTiles) {
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    uint8_t *b = reinterpret_cast<uint8_t *>(s.b) + off;
    *reinterpret_cast<uint4 *>(b) = cand ? ph : z;
    *reinterpret_cast<uint4 *>(b + T3_B_PART) = cand ? pl : z;
  }
  s_sq[c][lane] = sq;
  __syncthreads();
  if (c == 0) {
    float t = 0.0f;
#pragma unroll
    for (int i = 0; i < 16; i++) t += s_sq[i][lane];
    float nrm = sqrtf(t) * 1.0001f;
    if (row < s.n) s.norms[row] = nrm;
    if (cand) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) nrm = fmaxf(nrm, __shfl_xor_sync(0xffffffffu, nrm, o));
      if (lane == 0) atomicMax(reinterpret_cast<int *>(s.bmax), __float_as_int(nrm));
    }
    if (lane == 0 && s_bad) atomicMax(reinterpret_cast<int *>(gate), 1);
  }
}

// Unit u of the GEMM: its table tile, its A and B operand tiles (in a16 / b16), its candidate tile nt in the direction,
// and whether it is the last unit of its row tile.  A call has one direction, its tiles in row-tile order; a batch wave
// (TABLE) has a table of directions, d the one of the previous unit (the units only grow).
struct T3Unit {
  int gt, aTile, bTile, nt;
  bool last;
};
template <bool TABLE>
__device__ __forceinline__ T3Unit t3_unit(const TcPlan &pl, const MbDir *__restrict__ dirs, int numDirs, int &d, int u)
{
  T3Unit r;
  if (TABLE) {
    while (d + 1 < numDirs && dirs[d + 1].u0 <= u) d++;
    const int n_nt = dirs[d].n_nt, l = u - dirs[d].u0, mt = l / n_nt;
    r.nt = l - mt * n_nt;
    r.gt = dirs[d].gt0 + mt; r.aTile = dirs[d].aTile0 + mt; r.bTile = dirs[d].bTile0 + r.nt;
    r.last = r.nt == n_nt - 1;
  } else {
    const int mt = u / pl.n_nt;
    r.nt = u - mt * pl.n_nt;
    r.gt = r.aTile = mt; r.bTile = r.nt;
    r.last = (u + 1) / pl.n_nt != mt;
  }
  return r;
}

template <bool TABLE>
__global__ void __launch_bounds__(T3_THREADS, 1)
t3_gemm_kernel(const TcPlan pl, const T3Buffers bf, const MbDir *__restrict__ dirs, int numDirs)
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
    mbarrier_init(&bar_a_full, 1); mbarrier_init(&bar_a_empty, 8);
    for (int s = 0; s < T3_STAGES; s++) { mbarrier_init(&bar_b_full[s], 1); mbarrier_init(&bar_b_empty[s], 8); }
    mbarrier_init_fence();
  }
  __syncthreads();

  if (warp == 0) {
    // ============================ producer: bulk copies of whole operand tiles ============================
    if (lane == 0) {
      int runIdx = 0, prevGt = -1;
      int d = TABLE ? table_find(dirs, numDirs, &MbDir::u0, u_begin) : 0;
      for (int u = u_begin, i = 0; u < u_end; u++, i++) {
        const T3Unit un = t3_unit<TABLE>(pl, dirs, numDirs, d, u);
        if (un.gt != prevGt) {
          // every MMA of the previous run must have read the A tile before it is overwritten
          if (runIdx > 0) mbarrier_wait(&bar_a_empty, (runIdx - 1) & 1);
          mbarrier_expect_tx(&bar_a_full, T3_A_BYTES);
          bulk_g2s(sA, reinterpret_cast<const uint8_t *>(bf.a16) + (size_t)un.aTile * T3_A_BYTES, T3_A_BYTES,
                   &bar_a_full);
          prevGt = un.gt; runIdx++;
        }
        const int s = i % T3_STAGES, it = i / T3_STAGES;
        if (it > 0) mbarrier_wait(&bar_b_empty[s], (it - 1) & 1);
        mbarrier_expect_tx(&bar_b_full[s], T3_B_BYTES);
        bulk_g2s(sB + s * T3_B_BYTES, reinterpret_cast<const uint8_t *>(bf.b16) + (size_t)un.bTile * T3_B_BYTES,
                 T3_B_BYTES, &bar_b_full[s]);
      }
    }
  } else if (warp >= 4) {
    // ============================ consumers: MMAs and top-3 tables, one warpgroup per 64 rows ============================
    const unsigned int FULL = 0xffffffffu;
    const int g = (warp - 4) >> 2, wi = warp & 3;
    const int hb = (lane >> 1) & 1;       // this lane's 4-candidate groups are those of the partitions of parity hb
    const int rowInTile = g * T3_M + 16 * wi + (lane >> 2);   // and +8 (accumulator fragment rows)
    const uint32_t aBase = smem_addr(sA) + g * T3_M * 16, bBase = smem_addr(sB);
    float acc[64];
#pragma unroll
    for (int e = 0; e < 64; e++) acc[e] = 0.0f;
    // [fragment row][partition 2q + hb]
    float g1[2][4], g2[2][4], g3[2][4];
    int i1[2][4], i2[2][4];
    int prevGt = -1, runIdx = 0;
    int d = TABLE ? table_find(dirs, numDirs, &MbDir::u0, u_begin) : 0;
    size_t slot = 0;
    for (int u = u_begin, i = 0; u < u_end; u++, i++) {
      const T3Unit un = t3_unit<TABLE>(pl, dirs, numDirs, d, u);
      if (un.gt != prevGt) {
        slot = tc_slot(un.gt, cta, rowInTile);
        mbarrier_wait(&bar_a_full, runIdx & 1);
        prevGt = un.gt; runIdx++;
#pragma unroll
        for (int r = 0; r < 2; r++)
#pragma unroll
          for (int q = 0; q < 4; q++) { g1[r][q] = 0.0f; g2[r][q] = 0.0f; g3[r][q] = 0.0f; i1[r][q] = -1; i2[r][q] = -1; }
      }
      const int s = i % T3_STAGES, it = i / T3_STAGES;
      mbarrier_wait(&bar_b_full[s], it & 1);
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
      const bool lastOfRun = (u + 1 == u_end) || un.last;
      if (lane == 0) {
        mbarrier_arrive(&bar_b_empty[s]);
        if (lastOfRun) mbarrier_arrive(&bar_a_empty);
      }
      // columns 8j + 2(lane % 4) + {0, 1}: the lane pair (lane, lane ^ 1) holds group 2j + hb of partition 2(j % 4) + hb
      const int gbase = un.nt * (T3_N / 4) + hb;
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
// Eight lanes per row (four rows per warp): merge the segments' top-3 tables (lane = partition), decide which partitions
// can matter, re-score their first (and, within delta, second) groups exactly (lane = candidate, eight per round), then
// the rule's final step.  Two rules share every step but the threshold pool, the certification and the final step:
// - the reference rule (MatchSiftData): the reference's per-partition rule (matching.cu:354-359, stated
//   order-independently) and 8-way merge (:378-390) into set 1's five match fields;
// - KNN: the true two nearest neighbours (match_knn.cu states the order) among all n2 candidates.  Per partition the
//   merged tables give G >= S >= Th and the groups I1, I2.  T is the second largest of the 16 values {G[0..7], S[0..7]}:
//   two distinct groups have approximate maxima >= T, so two distinct candidates have exact scores >= T - eps, and
//   score2 >= T - eps.  A candidate whose group is not re-scored lies in a group below T - delta (delta = 2 eps): it is
//   either a partition's third group or lower (<= Th, certified < T - delta) or an I1 / I2 group below T - delta.  Its
//   exact score is then < T - eps <= score2, strictly, so the top two of the re-scored candidates (at most 8 x 2 groups
//   x 4 = T3_TAB) are the row's top two, ties included.  T > 2 delta keeps both clearly positive.
#define T3_RW 4                       // warps per CTA (16 rows)
#define T3_TAB 64                     // exact scores a row can collect (8 partitions x 2 groups x 4)

struct T3ResolveXy {
  float2 xy[T3_RW][4][T3_TAB];        // the candidates' positions (match_xpos / match_ypos)
};
struct T3ResolveNoXy {};
// Only the reference rule carries positions: the top-2 rule keeps the smaller footprint and its resident CTAs.
template <bool KNN>
struct T3ResolveSmem : std::conditional_t<KNN, T3ResolveNoXy, T3ResolveXy> {
  float4 a[T3_RW][4][33];             // the rows' own descriptors (+1: the four rows of a warp hit different banks)
  float sc[T3_RW][4][T3_TAB];         // exact scores
  int p2[T3_RW][4][T3_TAB];           // their indices
  int grp[T3_RW][4][16];              // candidate group list
};

// neighbour order: larger score first, then the lower index; the empty entry (0, -1) is passed by positive scores only
__device__ __forceinline__ void knn_top2_insert(float &s1, int &j1, float &s2, int &j2, float s, int j)
{
  if (s > s1 || (s == s1 && j < j1)) { s2 = s1; j2 = j1; s1 = s; j1 = j; }
  else if (s > s2 || (s == s2 && j < j2)) { s2 = s; j2 = j; }
}

// A call resolves one direction, `one`, and lists its uncertified rows in bf.fbRows.  A batch wave (TABLE, top-2 rule)
// resolves every direction of the table, each with ceil(n1 / 16) CTAs from its cta0 on; its rows go to the fallback as
// {direction, row} entries (cap of them), all of them when either set raised its bad-input flag.
template <bool KNN, bool TABLE>
__global__ void __launch_bounds__(32 * T3_RW)
t3_resolve_kernel(const TcPlan pl, const T3Buffers bf, const MbDir one, const MbDir *__restrict__ dirs, int numDirs,
                  int2 *__restrict__ entries, unsigned int *__restrict__ numEntries, int cap)
{
  static_assert(KNN || !TABLE, "a batch wave runs the top-2 rule");
  __shared__ T3ResolveSmem<KNN> sm;
  __shared__ unsigned int s_chains;      // one global atomic per CTA: same-address atomics serialise in L2
  if (threadIdx.x == 0) s_chains = 0;
  __syncthreads();
  const unsigned int FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int sub = lane >> 3, p = lane & 7;                   // row within the warp; partition / candidate slot
  int blk = blockIdx.x, dir = 0;
  MbDir D = one;
  if (TABLE) {
    dir = table_find(dirs, numDirs, &MbDir::cta0, (int)blockIdx.x);
    D = dirs[dir];
    blk -= D.cta0;
  }
  const int row = (blk * T3_RW + w) * 4 + sub;
  const bool valid = row < D.n1;
  if constexpr (TABLE) {
    if (*D.bad1 | *D.bad2) {                                  // gated: every row takes the exact way
      if (valid && p == 0) {
        atomicAdd(&D.counters[0], 1u);
        const unsigned e = atomicAdd(numEntries, 1u);
        if (e < (unsigned)cap) entries[e] = make_int2(dir, row);
      }
      return;
    }
  }
  const int rrow = valid ? row : D.n1 - 1;                    // clamped: padding lanes mirror the last row
  const int mt = rrow / T3_MT, rowInTile = rrow - mt * T3_MT;
  // the row's descriptor (each lane four float4), needed by every chain
#pragma unroll
  for (int j = 0; j < 4; j++) sm.a[w][sub][p + 8 * j] = __ldg(reinterpret_cast<const float4 *>(D.s1[rrow].data) + p + 8 * j);
  const float bmax = __int_as_float(*reinterpret_cast<const int *>(D.bmax));
  const float normA = D.norms[rrow];
  // merged top-3 of partition p.  The segments' tables are fetched together (independent loads, one
  // round trip) and inserted afterwards; T3_SEG bounds the unrolled part, more segments take the loop.
  float G = 0.0f, S = 0.0f, Th = 0.0f;
  int I1 = -1, I2 = -1;
  {
    const int gt = D.gt0 + mt;
    const int u0 = D.u0 + mt * D.n_nt, u1 = u0 + D.n_nt - 1;
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
        const float *q = bf.pm + tc_slot(gt, c, rowInTile) * T3_PM;
        v[k][0] = q[p]; v[k][1] = q[8 + p]; v[k][2] = q[16 + p];
        id[k][0] = __float_as_int(q[24 + p]); id[k][1] = __float_as_int(q[32 + p]);
      } else {
        v[k][0] = v[k][1] = v[k][2] = 0.0f; id[k][0] = id[k][1] = -1;
      }
    }
#pragma unroll
    for (int k = 0; k < T3_SEG; k++) { insert(v[k][0], id[k][0]); insert(v[k][1], id[k][1]); insert(v[k][2], -1); }
    for (int c = c0 + T3_SEG; c <= c1; c++) {
      const float *q = bf.pm + tc_slot(gt, c, rowInTile) * T3_PM;
      insert(q[p], __float_as_int(q[24 + p])); insert(q[8 + p], __float_as_int(q[32 + p])); insert(q[16 + p], -1);
    }
    G *= T3_UNSCALE; S *= T3_UNSCALE; Th *= T3_UNSCALE;
  }
  const float delta = 2.0f * (T3_C1 * normA * bmax + T3_C2 * (normA + bmax));
  // m2 = the second largest element of the rule's pool
  float m1 = 0.0f, m2 = 0.0f;
  if constexpr (KNN) {
    // T: {G[0..7], S[0..7]}
#pragma unroll
    for (int y = 0; y < 8; y++) {
      const float gy = __shfl_sync(FULL, G, y, 8), sy = __shfl_sync(FULL, S, y, 8);
      m2 = fmaxf(m2, fminf(m1, gy));
      m1 = fmaxf(m1, gy);
      m2 = fmaxf(m2, fminf(m1, sy));
      m1 = fmaxf(m1, sy);
    }
  } else {
    // L: {G[0..7], S[0]} (S[0] bounds partition 0's second best, quirk Q9)
    m1 = __shfl_sync(FULL, S, 0, 8);
#pragma unroll
    for (int y = 0; y < 8; y++) {
      const float gy = __shfl_sync(FULL, G, y, 8);
      m2 = fmaxf(m2, fminf(m1, gy));
      m1 = fmaxf(m1, gy);
    }
  }
  const bool rowOk = (m2 > 2.0f * delta) && (m2 < 3.0e38f);    // the deciding elements are clearly positive
  bool cert, use1, use2;
  if constexpr (KNN) {
    const float low = m2 - delta;
    cert = Th <= 0.0f || Th < low;
    use1 = rowOk && I1 >= 0 && G >= low;
    use2 = rowOk && I2 >= 0 && S >= low;
  } else {
    const float L = m2;
    const bool rel = rowOk && (G >= L - delta);
    const float low = (p == 0 ? fminf(L, G) : G) - delta;      // partition 0 also supplies its second best
    cert = !rel || Th <= 0.0f || Th < low;
    use1 = rel && I1 >= 0;
    use2 = rel && I2 >= 0 && S >= low;
  }
  const unsigned int certMask = (__ballot_sync(FULL, cert) >> (8 * sub)) & 0xffu;
  const bool ok = valid && rowOk && certMask == 0xffu;
  if (valid && !ok && p == 0) {
    const unsigned at = atomicAdd(&D.counters[0], 1u);
    if (TABLE) {
      const unsigned e = atomicAdd(numEntries, 1u);
      if (e < (unsigned)cap) entries[e] = make_int2(dir, row);
    } else if (at < (unsigned)pl.n_mt * T3_MT) {
      // every row lists itself at most once, so the index stays below n1 when the counter started at zero; the clamp
      // keeps a stale counter (a previous call that failed half-way) from writing past the list
      bf.fbRows[at] = row;
    }
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
      // candidates past n2 (zero rows of the last tile, top-2 rule) score 0: never a neighbour.  In the reference rule
      // the B operand is zero from n2v = 32*floor(n2/32) on, so such groups never enter the tables.
      float acc = 0.0f;
      float2 xy = make_float2(0.0f, 0.0f);
      if (p2 < D.n2) {
        const float4 *bp = reinterpret_cast<const float4 *>(D.s2[p2].data);
        if constexpr (!KNN) xy = make_float2(D.s2[p2].xpos, D.s2[p2].ypos);
        // the reference's score: sequential k = 0..127 FMA chain starting from 0 (matching.cu:338-351).
        // Software pipeline: the next eight float4 of the candidate are in flight while eight are consumed.
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
      }
      sm.sc[w][sub][c] = acc;
      sm.p2[w][sub][c] = p2;
      if constexpr (!KNN) sm.xy[w][sub][c] = xy;
    }
  }
  __syncwarp();
  if constexpr (KNN) {
    // lane p: top two of entries p, p + 8, ...; then a butterfly over the row's eight lanes (the order is total)
    float s1 = 0.0f, s2 = 0.0f;
    int j1 = -1, j2 = -1;
    for (int e = p; e < ncand; e += 8) knn_top2_insert(s1, j1, s2, j2, sm.sc[w][sub][e], sm.p2[w][sub][e]);
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) {
      const float t1 = __shfl_xor_sync(FULL, s1, o, 8), t2 = __shfl_xor_sync(FULL, s2, o, 8);
      const int k1 = __shfl_xor_sync(FULL, j1, o, 8), k2 = __shfl_xor_sync(FULL, j2, o, 8);
      knn_top2_insert(s1, j1, s2, j2, t1, k1);
      knn_top2_insert(s1, j1, s2, j2, t2, k2);
    }
    if (ok && p == 0) {
      D.idx[row] = make_int2(j1, j2);
      D.score[row] = make_float2(s1, s2);
    }
  } else {
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
      SiftPoint *o = const_cast<SiftPoint *>(D.s1) + row;     // a match writes set 1's match fields in place
      const float2 xy = ent >= 0 ? sm.xy[w][sub][ent] : make_float2(0.0f, 0.0f);
      o->score = mx;
      o->match = idx;
      o->match_xpos = xy.x;
      o->match_ypos = xy.y;
      o->ambiguity = __fdiv_rn(sec, __fadd_rn(mx, 1e-6f));
    }
  }
  if (ok && p == 0) atomicAdd(&s_chains, (unsigned)ncand);
  __syncthreads();
  if (threadIdx.x == 0 && s_chains) { atomicAdd(&D.counters[1], s_chains >> 2); atomicAdd(&D.counters[2], s_chains); }
}

// exact SIMT scan of the rows the tensor path could not certify (match.cu)
int match_exact_fallback(SiftPoint *s1, int n1, const SiftPoint *s2, int n2, const int *rows, const unsigned int *nrows,
                         const unsigned int *gate, cudaStream_t st);

// ------------------------------------------------------------------------------ host
bool match_tensor_supported()
{
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return false;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  return major == 9;
}

// persistent GEMM schedule of `total` units: at most one CTA per SM, U units each
static void t3_schedule(TcPlan &pl, int sms)
{
  pl.grid = pl.total < sms ? pl.total : sms;
  pl.U = idivup(pl.total, pl.grid);
  pl.grid = idivup(pl.total, pl.U);
}
// n1 rows against the first n2v candidates
static TcPlan t3_plan(int n1, int n2v, int sms)
{
  TcPlan pl;
  pl.n_mt = idivup(n1, T3_MT); pl.n_nt = idivup(n2v, T3_N);
  pl.total = pl.n_mt * pl.n_nt;
  t3_schedule(pl, sms);
  return pl;
}
// top-3 table slots of `tiles` row tiles run by `grid` CTAs (tc_slot)
static size_t t3_slots(int tiles, int grid) { return ((size_t)tiles + grid) * T3_MT; }
static size_t t3_slots(const TcPlan &pl) { return t3_slots(pl.n_mt, pl.grid); }

// A tensor-path call once its prep kernel is in: each direction's plan, view of the workspace and resolve view (its
// rows, candidates, norms, counters; a knn call adds the neighbour lists), the bad-input gate (shared: any bad value,
// either set), the call's flag area and the timing events (or null).
struct T3Call {
  TcPlan pf, pr;
  T3Buffers fw, rv;
  MbDir df, dr;
  const unsigned int *gate;
  const float *flags;
  cudaEvent_t *tev;
};

// The part of a call that matching and knn share: grows the workspace, fills the prep sets, builds the forward view
// (set 1 against set 2) and, with both, the reverse one, and launches the prep kernel.  n1v / n2v are the rows of each
// set that are candidates of the other direction: 32*floor(n/32) in a match (quirk Q7), all of them in knn.  Set 1 has
// the A role, set 2 the B role, and with both each set has both roles.  Workspace: the sets' tiles one after the other
// in tcA (their norms likewise in tcNorms, set 2's unread in a one-way call), the B-role copies in tcB.  The top-3 tables
// and the fallback row list are shared: the two directions are stream-ordered.  Flags and counters live in two 64-byte
// areas used alternately: a call's prep kernel clears the other one for the next call, which saves a memset node.
static int t3_setup(DeviceCtx &c, const SiftPoint *s1, int n1, int n1v, const SiftPoint *s2, int n2, int n2v, bool both,
                    T3Call &t)
{
  t.pf = t3_plan(n1, n2v, c.sms);
  t.pr = both ? t3_plan(n2, n1v, c.sms) : TcPlan{};
  T3PrepSet p[2] = {{s1, n1, both ? n1v : 0}, {s2, both ? n2 : n2v, n2v}};
  size_t aOff[2], bOff[2], nOff[2], aBytes = 0, bBytes = 0, rows = 0;
  bool copy[2];
  for (int k = 0; k < 2; k++) {
    const int tiles = idivup(p[k].n, T3_MT);
    p[k].blocks = tiles * (T3_MT / 32);
    p[k].bTiles = idivup(p[k].nv, T3_N);
    aOff[k] = aBytes; aBytes += (size_t)tiles * T3_A_BYTES;
    nOff[k] = rows; rows += (size_t)tiles * T3_MT;
    // a set needs its own B-role copy when its tail rows [nv, n) lie in a tile that the B role reads (never in knn)
    copy[k] = p[k].n != p[k].nv && p[k].nv % T3_N != 0;
    bOff[k] = bBytes; bBytes += copy[k] ? (size_t)p[k].bTiles * T3_B_BYTES : 0;
  }
  const size_t slots = t3_slots(t.pf) > t3_slots(t.pr) ? t3_slots(t.pf) : t3_slots(t.pr);
  const size_t fbRows = (size_t)(t.pf.n_mt > t.pr.n_mt ? t.pf.n_mt : t.pr.n_mt) * T3_MT;
  const cudaStream_t st = c.stream;
  int r;
  if ((r = c.tcA.grow(aBytes)) < 0 || (r = c.tcB.grow(bBytes)) < 0 || (r = c.tcNorms.grow(rows * sizeof(float))) < 0 ||
      (r = c.tcTables.grow(slots * T3_PM * sizeof(float))) < 0 || (r = c.tcRows.grow(fbRows * sizeof(int))) < 0)
    return r;
  if (!c.tcFlags.p) {
    if ((r = c.tcFlags.grow(128)) < 0) return r;
    CS_CUDA(cudaMemsetAsync(c.tcFlags.p, 0, 128, st));
  }
  float *flags = c.tcFlags.as<float>() + 16 * (c.tcCalls & 1);
  float *nextFlags = c.tcFlags.as<float>() + 16 * ((c.tcCalls + 1) & 1);
  if (c.tcDirty) CS_CUDA(cudaMemsetAsync(c.tcFlags.p, 0, 128, st));   // a previous call failed between its launches
  c.tcDirty = true;                                                  // until this call's launches are all in
  if (!c.tcConfigured) {
    CS_CUDA(cudaFuncSetAttribute(t3_gemm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, T3_SMEM_BYTES));
    c.tcConfigured = true;
  }
  auto at = [](void *base, size_t bytes) { return reinterpret_cast<__half *>(static_cast<uint8_t *>(base) + bytes); };
  for (int k = 0; k < 2; k++) {
    p[k].a = at(c.tcA.p, aOff[k]);
    p[k].b = copy[k] ? at(c.tcB.p, bOff[k]) : nullptr;
    p[k].norms = c.tcNorms.as<float>() + nOff[k];
  }
  // flags [0] / [2] take the candidates' max norm of the forward / reverse direction, i.e. of set 2 / set 1; the
  // counters of the two directions are flags [4..6] and [8..10]
  p[0].bmax = flags + 2; p[1].bmax = flags;
  unsigned int *counters = reinterpret_cast<unsigned int *>(flags);
  t.fw = {p[0].a, copy[1] ? p[1].b : p[1].a, c.tcTables.as<float>(), c.tcRows.as<int>()};
  t.rv = {p[1].a, copy[0] ? p[0].b : p[0].a, c.tcTables.as<float>(), c.tcRows.as<int>()};
  auto view = [](const SiftPoint *a, int na, const SiftPoint *b, int nb, const float *norms, const float *bmax,
                 unsigned int *cnt, int n_nt) {
    MbDir d{};
    d.s1 = a; d.s2 = b; d.n1 = na; d.n2 = nb;
    d.norms = norms; d.bmax = bmax; d.counters = cnt; d.n_nt = n_nt;
    return d;
  };
  t.df = view(s1, n1, s2, n2, p[0].norms, flags, counters + 4, t.pf.n_nt);
  t.dr = view(s2, n2, s1, n1, p[1].norms, flags + 2, counters + 8, t.pr.n_nt);
  t.gate = counters + 1;
  t.flags = flags;
  t.tev = match_timing_events();
  if (t.tev) cudaEventRecord(t.tev[0], st);
  t3_prep_kernel<false><<<p[0].blocks + p[1].blocks, 512, 0, st>>>(p[0], p[1], nullptr, 0, flags + 1, nextFlags);
  count_launch();
  CS_CUDA(cudaGetLastError());
  if (t.tev) cudaEventRecord(t.tev[1], st);
  return 0;
}

// exact two-nearest-neighbour scan of the listed rows, or of every row if *gate != 0 (match_knn.cu)
int knn_exact_fallback(DeviceCtx &c, const SiftPoint *s1, int n1, const SiftPoint *s2, int n2, int *idx, float *score,
                       const int *rows, const unsigned int *nrows, const unsigned int *gate);

// One direction after the prep kernel: GEMM, resolve, then the rule's exact kernel for the rows that could not be
// certified -- or, for inputs the split cannot bound (*gate != 0: |x| >= 8, NaN, Inf), for every row; which of the two
// is decided on the device.  KNN: the two nearest neighbours into d.idx / d.score; else the reference rule into set 1's
// match fields.  ev (optional): three events, recorded after each launch.
template <bool KNN>
static int t3_direction(DeviceCtx &c, const TcPlan &pl, const T3Buffers &bf, const MbDir &d, const unsigned int *gate,
                        cudaEvent_t *ev)
{
  const cudaStream_t st = c.stream;
  t3_gemm_kernel<false><<<pl.grid, T3_THREADS, T3_SMEM_BYTES, st>>>(pl, bf, nullptr, 0);
  if (ev) cudaEventRecord(ev[0], st);
  t3_resolve_kernel<KNN, false><<<idivup(d.n1, 4 * T3_RW), 32 * T3_RW, 0, st>>>(pl, bf, d, nullptr, 0, nullptr, nullptr, 0);
  if (ev) cudaEventRecord(ev[1], st);
  count_launch(2);
  CS_CUDA(cudaGetLastError());
  const int r = KNN ? knn_exact_fallback(c, d.s1, d.n1, d.s2, d.n2, reinterpret_cast<int *>(d.idx),
                                         reinterpret_cast<float *>(d.score), bf.fbRows, d.counters, gate)
                    : match_exact_fallback(const_cast<SiftPoint *>(d.s1), d.n1, d.s2, d.n2, bf.fbRows, d.counters, gate,
                                           st);
  if (r < 0) return r;
  if (ev) cudaEventRecord(ev[2], st);
  return 0;
}

// the call's counters to the host, read by match_tensor_stats() after the caller's synchronize
static int t3_end(DeviceCtx &c, const float *flags)
{
  CS_CUDA(cudaMemcpyAsync(c.h_tcFlags, flags, 64, cudaMemcpyDeviceToHost, c.stream));
  c.tcCalls++;                          // the prep kernel of this call cleared the other flag area for the next one
  c.tcDirty = false;
  c.tcPendingStats = true;
  return 0;
}

// the stages of a tensor-path call; a one-way call has the first 4, a two-way knn call 7, a mutual call 8
static const char *const t3_stages[] = {"prep", "gemm", "resolve", "exact-fallback", "reverse-gemm", "reverse-resolve",
                                        "reverse-exact-fallback", "pairs"};

// Set 1's five match fields; with mu (32 or more rows in each set) also set 2's, exactly as a one-way match of set 2
// against set 1 writes them, then the cross-checked pairs (launch_mutual_pairs).  One prep launch converts each set once
// for every role it has (T3PrepSet); each direction then runs on its own plan and its own view of the workspace.
int match_tensor(DeviceCtx &c, SiftPoint *s1, int n1, SiftPoint *s2, int n2, const MutualArgs *mu)
{
  const int n1v = (n1 / 32) * 32, n2v = (n2 / 32) * 32;   // matching.cu:325 (quirk Q7)
  if (!mu) {
    if (n1 <= 0) return 0;
    if (n2v == 0 || !match_tensor_supported()) return match_exact(s1, n1, s2, n2, c.stream);
  } else if (n1v == 0 || n2v == 0) {
    set_error("match_tensor: a mutual match needs 32 rows or more in each set");
    return CS_E_ARG;
  }
  T3Call t;
  int r;
  if ((r = t3_setup(c, s1, n1, n1v, s2, n2, n2v, mu != nullptr, t)) < 0) return r;
  cudaEvent_t *tev = t.tev;
  if ((r = t3_direction<false>(c, t.pf, t.fw, t.df, t.gate, tev ? tev + 2 : nullptr)) < 0) return r;
  if (mu) {
    if ((r = t3_direction<false>(c, t.pr, t.rv, t.dr, t.gate, tev ? tev + 5 : nullptr)) < 0) return r;
    if ((r = launch_mutual_pairs(c, s1, n1, s2, n2, *mu)) < 0) return r;
    if (tev) cudaEventRecord(tev[8], c.stream);
  }
  if (tev) report_stage_times(tev, t3_stages, mu ? 8 : 4, "%s timing %dx%d", mu ? "mutual" : "match", n1, n2);
  return t3_end(c, t.flags);
}

// The two nearest neighbours of every row of set 1 among all n2 candidates (idx1 / score1, [n1][2]); with idx2 also
// those of every row of set 2 among set 1's n1 rows.  The records are only read.  Same setup as match_tensor; there is
// no Q7 tail, so each set's A tiles are also the other direction's B operand (rows past n are zeros, score 0, and never
// enter the tables).
int match_knn_tensor(DeviceCtx &c, const SiftPoint *s1, int n1, const SiftPoint *s2, int n2, int *idx1, float *score1,
                     int *idx2, float *score2)
{
  if (n1 <= 0 || n2 <= 0) return 0;
  const bool both = idx2 != nullptr;
  T3Call t;
  int r;
  if ((r = t3_setup(c, s1, n1, n1, s2, n2, n2, both, t)) < 0) return r;
  cudaEvent_t *tev = t.tev;
  t.df.idx = reinterpret_cast<int2 *>(idx1); t.df.score = reinterpret_cast<float2 *>(score1);
  t.dr.idx = reinterpret_cast<int2 *>(idx2); t.dr.score = reinterpret_cast<float2 *>(score2);
  if ((r = t3_direction<true>(c, t.pf, t.fw, t.df, t.gate, tev ? tev + 2 : nullptr)) < 0) return r;
  if (both && (r = t3_direction<true>(c, t.pr, t.rv, t.dr, t.gate, tev ? tev + 5 : nullptr)) < 0) return r;
  if (tev) report_stage_times(tev, t3_stages, both ? 7 : 4, "knn timing %dx%d", n1, n2);
  return t3_end(c, t.flags);
}

// statistics of the last tensor-path call on this context (call after the stream was synchronized);
// a two-way call reports both directions summed
void match_tensor_stats(DeviceCtx &c, unsigned long long stats[4])
{
  if (!c.tcPendingStats) return;
  c.tcPendingStats = false;
  const unsigned int *h = c.h_tcFlags;
  if (h[1] != 0) { stats[0] = stats[1] = 0; stats[2] = ~0ull; return; }   // everything went the exact way
  stats[0] = (unsigned long long)h[4 + 1] + h[8 + 1];                     // [8..10] stay zero in a single direction
  stats[1] = (unsigned long long)h[4 + 2] + h[8 + 2];
  stats[2] = (unsigned long long)h[4 + 0] + h[8 + 0];
}

// ------------------------------------------------------------------------------ batched knn directions
// A wave (cs_match_ratio_batch states the rule): consecutive non-empty jobs whose scratch -- per distinct set its
// operand tiles and norms, per direction its top-3 tables, neighbour lists and fallback entries -- fits WAVE_BYTES.
// Every wave runs the same four launches (prep, GEMM, knn resolve, list fallback), then the caller's last step:
// ratio flags and pair writes for cs_match_ratio_batch, the word copy for cs_vocab_assign.
static size_t mb_set_bytes(int n) { return (size_t)idivup(n, T3_MT) * T3_MT * (T3_A_BYTES / T3_MT + sizeof(float)); }
static size_t mb_dir_bytes(int n1)
{
  return (size_t)idivup(n1, T3_MT) * T3_MT * T3_PM * sizeof(float) + (size_t)n1 * (sizeof(int2) + sizeof(float2) + sizeof(int2));
}

struct MbWave {
  std::vector<int> jobs;            // the jobs, in order
  std::vector<int> sets;            // the distinct sets, in order of first use
  int dirs = 0, tiles = 0, dirTiles = 0, rows = 0, words = 0, pairCtas = 0, units = 0, resolveCtas = 0, prepCtas = 0;
  size_t bytes = 0;                 // the rule's scratch
  size_t zeroWords = 0;
  // The wave's pinBytes in c.h_mb, from pinOff: the tables (sets at 0, directions at dirsAt, jobs at jobsAt; uploaded
  // to c.mbTables), then from stateAt the state's zeroWords (copied back).  Every piece starts at a multiple of 16 bytes.
  size_t pinOff = 0, pinBytes = 0, dirsAt = 0, jobsAt = 0, stateAt = 0;
};

static std::vector<MbWave> mb_waves(const cs_match_set *sets, int numSets, const cs_match_job *jobs, int numJobs,
                                    bool cross)
{
  std::vector<MbWave> waves;
  std::vector<int> mark((size_t)numSets, -1);             // the last wave that converts the set
  for (int p = 0; p < numJobs; p++) {
    const int a = jobs[p].set1, b = jobs[p].set2, na = sets[a].n, nb = sets[b].n;
    if (na == 0 || nb == 0) continue;
    auto cost = [&](int w) {
      size_t x = mb_dir_bytes(na) + (cross ? mb_dir_bytes(nb) : 0);
      if (mark[a] != w) x += mb_set_bytes(na);
      if (b != a && mark[b] != w) x += mb_set_bytes(nb);
      return x;
    };
    int w = (int)waves.size() - 1;
    if (w < 0 || waves[w].bytes + cost(w) > WAVE_BYTES) { waves.emplace_back(); w++; }
    MbWave &v = waves[w];
    v.bytes += cost(w);
    for (int s : {a, b})
      if (mark[s] != w) {
        mark[s] = w;
        v.sets.push_back(s);
        v.tiles += idivup(sets[s].n, T3_MT);
        v.prepCtas += idivup(sets[s].n, T3_MT) * (T3_MT / 32);
      }
    v.jobs.push_back(p);
    for (int k = 0; k < (cross ? 2 : 1); k++) {
      const int n1 = k ? nb : na, n2 = k ? na : nb;
      v.dirs++;
      v.dirTiles += idivup(n1, T3_MT);
      v.units += idivup(n1, T3_MT) * idivup(n2, T3_N);
      v.resolveCtas += idivup(n1, 4 * T3_RW);
      v.rows += n1;
    }
    v.words += list_words(na);
    v.pairCtas += list_ctas(na);
  }
  size_t pin = 0;
  for (MbWave &v : waves) {
    const size_t S = v.sets.size(), D = v.dirs, J = v.jobs.size();
    v.zeroWords = (2 * S + 4 * D + J + 1 + 3) & ~(size_t)3;
    Layout L(16);
    L.take(S * sizeof(T3PrepSet));
    v.dirsAt = L.take(D * sizeof(MbDir));
    v.jobsAt = L.take(J * sizeof(PairJob));
    v.stateAt = L.take(v.zeroWords * sizeof(unsigned int));
    v.pinOff = pin;
    v.pinBytes = L.bytes;
    pin += v.pinBytes;
  }
  return waves;
}

// The device tables of a wave in pinned memory, with pointers into the context's buffers; out[p] for its jobs.
// Device state: [2 s] set s's max norm, [2 s + 1] its bad-input flag; [2 S + 4 d] direction d's counters; then each
// job's pair total and the fallback entry count (all cleared per wave); then the ballot words and CTA counts.
static void mb_fill(DeviceCtx &c, const MbWave &v, const cs_match_set *sets, const cs_match_job *jobs, bool cross,
                    std::vector<int> &slot, RatioBatchOut *out)
{
  const int S = (int)v.sets.size(), D = v.dirs, J = (int)v.jobs.size();
  uint8_t *hp = c.h_mb.as<uint8_t>() + v.pinOff;
  T3PrepSet *hs = reinterpret_cast<T3PrepSet *>(hp);
  MbDir *hd = reinterpret_cast<MbDir *>(hp + v.dirsAt);
  PairJob *hj = reinterpret_cast<PairJob *>(hp + v.jobsAt);
  const unsigned int *hstate = reinterpret_cast<const unsigned int *>(hp + v.stateAt);
  unsigned int *st = c.mbState.as<unsigned int>();
  unsigned int *masks = st + v.zeroWords, *counts = masks + v.words;
  int2 *idx = c.mbLists.as<int2>();
  float2 *score = reinterpret_cast<float2 *>(idx + v.rows);
  int tile = 0, blk = 0;
  for (int k = 0; k < S; k++) {
    const cs_match_set &m = sets[v.sets[k]];
    slot[v.sets[k]] = k;
    T3PrepSet &p = hs[k];
    p = T3PrepSet{};
    p.pts = static_cast<const SiftPoint *>(m.pts);
    p.n = p.nv = m.n;
    p.blocks = idivup(m.n, T3_MT) * (T3_MT / 32);
    p.a = reinterpret_cast<__half *>(c.tcA.as<uint8_t>() + (size_t)tile * T3_A_BYTES);
    p.b = nullptr;
    p.norms = c.tcNorms.as<float>() + (size_t)tile * T3_MT;
    p.bmax = reinterpret_cast<float *>(st + 2 * k);
    p.bad = reinterpret_cast<float *>(st + 2 * k + 1);
    p.blk0 = blk;
    tile += idivup(m.n, T3_MT);
    blk += p.blocks;
  }
  int d = 0, u0 = 0, gt0 = 0, cta0 = 0, list0 = 0, word0 = 0, pcta0 = 0;
  for (int q = 0; q < J; q++) {
    const int pj = v.jobs[q];
    const cs_match_job &j = jobs[pj];
    const int a = slot[j.set1], b = slot[j.set2];
    int dd[2] = {-1, -1};
    for (int k = 0; k < (cross ? 2 : 1); k++, d++) {
      const int x = k ? b : a, y = k ? a : b;            // rows of set x against set y
      MbDir &r = hd[d];
      r.s1 = hs[x].pts; r.s2 = hs[y].pts; r.n1 = hs[x].n; r.n2 = hs[y].n;
      r.norms = hs[x].norms;
      r.bmax = hs[y].bmax;
      r.bad1 = reinterpret_cast<const unsigned int *>(hs[x].bad);
      r.bad2 = reinterpret_cast<const unsigned int *>(hs[y].bad);
      r.idx = idx + list0; r.score = score + list0;
      r.counters = st + 2 * S + 4 * d;
      r.aTile0 = hs[x].blk0 / (T3_MT / 32); r.bTile0 = hs[y].blk0 / (T3_MT / 32);
      r.n_nt = idivup(r.n2, T3_N);
      r.u0 = u0; r.gt0 = gt0; r.cta0 = cta0;
      u0 += idivup(r.n1, T3_MT) * r.n_nt; gt0 += idivup(r.n1, T3_MT); cta0 += idivup(r.n1, 4 * T3_RW);
      list0 += r.n1;
      dd[k] = d;
    }
    const MbDir &f = hd[dd[0]];
    PairJob &pjob = hj[q];
    pjob.jv = reinterpret_cast<const int *>(f.idx); pjob.jstride = 2;
    pjob.n1 = f.n1; pjob.n2 = f.n2;
    pjob.idx1 = f.idx; pjob.score1 = f.score;
    pjob.idx2 = cross ? hd[dd[1]].idx : nullptr; pjob.score2 = cross ? hd[dd[1]].score : nullptr;
    pjob.masks = masks + word0; pjob.blockCounts = counts + pcta0;
    pjob.pairs = reinterpret_cast<int2 *>(j.pairs); pjob.maxPairs = j.maxPairs;
    pjob.total = st + 2 * S + 4 * D + q;
    pjob.cta0 = pcta0;
    word0 += list_words(f.n1); pcta0 += list_ctas(f.n1);
    RatioBatchOut &o = out[pj];
    o.total = hstate + 2 * S + 4 * D + q;
    o.counters[0] = hstate + 2 * S + 4 * dd[0];
    o.counters[1] = cross ? hstate + 2 * S + 4 * dd[1] : nullptr;
    o.bad1 = hstate + 2 * a + 1; o.bad2 = hstate + 2 * b + 1;
  }
}

int ratio_batch_enqueue(DeviceCtx &c, const cs_match_set *sets, int numSets, const cs_match_job *jobs, int numJobs,
                        float maxRatio, float maxDistance, bool cross, RatioBatchOut *out)
{
  return knn_batch_enqueue(c, sets, numSets, jobs, numJobs, cross, out, "ratio-batch", "pairs", [&](const KnnWave &w) {
    return launch_ratio_pairs_batch(c, w.pairJobs, w.numJobs, w.pairCtas, maxRatio, maxDistance);
  });
}

int knn_batch_enqueue(DeviceCtx &c, const cs_match_set *sets, int numSets, const cs_match_job *jobs, int numJobs,
                      bool cross, RatioBatchOut *out, const char *name, const char *lastStage,
                      const KnnWaveFinish &finish)
{
  const std::vector<MbWave> waves = mb_waves(sets, numSets, jobs, numJobs, cross);
  if (waves.empty()) return 0;
  size_t tiles = 0, slots = 0, rows = 0, state = 0, tab = 0, pin = 0;
  for (const MbWave &v : waves) {
    tiles = std::max(tiles, (size_t)v.tiles);
    slots = std::max(slots, t3_slots(v.dirTiles, c.sms));
    rows = std::max(rows, (size_t)v.rows);
    state = std::max(state, v.zeroWords + v.words + v.pairCtas);
    tab = std::max(tab, v.stateAt);
    pin = v.pinOff + v.pinBytes;
  }
  const cudaStream_t st = c.stream;
  int r;
  if ((r = c.tcA.grow(tiles * T3_A_BYTES)) < 0 || (r = c.tcNorms.grow(tiles * T3_MT * sizeof(float))) < 0 ||
      (r = c.tcTables.grow(slots * T3_PM * sizeof(float))) < 0 || (r = c.mbTables.grow(tab)) < 0 ||
      (r = c.mbLists.grow(rows * (sizeof(int2) + sizeof(float2) + sizeof(int2)))) < 0 ||
      (r = c.mbState.grow(state * sizeof(unsigned int))) < 0)
    return r;
  if ((r = c.h_mb.grow(pin)) < 0) return r;
  if (!c.mbConfigured) {
    CS_CUDA(cudaFuncSetAttribute(t3_gemm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, T3_SMEM_BYTES));
    c.mbConfigured = true;
  }
  std::vector<int> slot((size_t)numSets, -1);
  cudaEvent_t *tev = match_timing_events();
  for (const MbWave &v : waves) {
    mb_fill(c, v, sets, jobs, cross, slot, out);
    const int S = (int)v.sets.size(), D = v.dirs, J = (int)v.jobs.size();
    uint8_t *hp = c.h_mb.as<uint8_t>() + v.pinOff;
    uint8_t *dt = c.mbTables.as<uint8_t>();
    const T3PrepSet *ds = reinterpret_cast<const T3PrepSet *>(dt);
    const MbDir *dd = reinterpret_cast<const MbDir *>(dt + v.dirsAt);
    const PairJob *dj = reinterpret_cast<const PairJob *>(dt + v.jobsAt);
    unsigned int *state = c.mbState.as<unsigned int>();
    int2 *entries = c.mbLists.as<int2>() + 2 * (size_t)v.rows;
    unsigned int *numEntries = state + 2 * S + 4 * D + J;
    TcPlan pl{};
    pl.total = v.units;
    t3_schedule(pl, c.sms);
    const T3Buffers bf = {c.tcA.as<__half>(), c.tcA.as<__half>(), c.tcTables.as<float>(), nullptr};
    CS_CUDA(cudaMemsetAsync(state, 0, v.zeroWords * sizeof(unsigned int), st));
    CS_CUDA(cudaMemcpyAsync(dt, hp, v.stateAt, cudaMemcpyHostToDevice, st));
    if (tev) cudaEventRecord(tev[0], st);
    t3_prep_kernel<true><<<v.prepCtas, 512, 0, st>>>(T3PrepSet{}, T3PrepSet{}, ds, S, nullptr, nullptr);
    if (tev) cudaEventRecord(tev[1], st);
    t3_gemm_kernel<true><<<pl.grid, T3_THREADS, T3_SMEM_BYTES, st>>>(pl, bf, dd, D);
    if (tev) cudaEventRecord(tev[2], st);
    t3_resolve_kernel<true, true><<<v.resolveCtas, 32 * T3_RW, 0, st>>>(pl, bf, MbDir{}, dd, D, entries, numEntries,
                                                                        v.rows);
    if (tev) cudaEventRecord(tev[3], st);
    count_launch(3);
    CS_CUDA(cudaGetLastError());
    if ((r = launch_knn_list_fallback(c, dd, entries, numEntries, v.rows)) < 0) return r;
    if (tev) cudaEventRecord(tev[4], st);
    const KnnWave w = {v.jobs, dj, J, v.pairCtas, c.mbLists.as<int2>(),
                       reinterpret_cast<const float2 *>(c.mbLists.as<int2>() + v.rows), v.rows};
    if ((r = finish(w)) < 0) return r;
    if (tev) cudaEventRecord(tev[5], st);
    CS_CUDA(cudaMemcpyAsync(hp + v.stateAt, state, v.zeroWords * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
    const char *const stages[] = {"prep", "gemm", "resolve", "exact-fallback", lastStage};
    if (tev) report_stage_times(tev, stages, 5, "%s timing %d jobs %d directions %d units", name, J, D, v.units);
  }
  return 0;
}

}  // namespace cs
