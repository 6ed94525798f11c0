// match_knn.cu -- exact FP32 two-nearest-neighbour search (the exact path of cs_match_knn2 / cs_match_ratio).
//
// Semantics: score(i, j) is the reference's score, the sequential k = 0..127 FMA chain starting from 0 (the same value
// MatchSiftData writes).  For every row i of set 1 all n2 candidates are visited (no quirk Q7 tail) and only scores
// > 0 count.  The two neighbours are the first two candidates in the total order (score descending, index ascending):
// j1 is the lowest index with the largest score, j2 the lowest index != j1 with the largest remaining score (it may
// equal score1).  A missing neighbour is index -1 with score 0.  This is COLMAP's brute-force loop (strict '>' in
// increasing j) with the second index kept as well.
//
// knn_exact_kernel is tiled like match_exact_kernel (32 rows x 32 candidates per step, 128 threads) and keeps top-2
// state per (row, thread); the candidate range is split over gridDim.y slices so that a handful of rows does not scan
// thousands of candidates in one CTA.  With more than one slice every slice writes its top two to a partial area and
// knn_merge_kernel combines them.  The merge key is a total order, so the result does not depend on the slicing.
#include "common.cuh"

namespace cs {

#define KX_ROWS 32          // rows of set 1 per CTA
#define KX_COLS 32          // candidates of set 2 per step
#define KX_LD 33            // row stride in float4 (+1 float4 padding: conflict-free LDS.128)
#define KX_THREADS 128
#define KX_MIN_STEPS 4      // candidate steps per slice at least (128 candidates)
#define KX_MAX_SLICES 128

// rows == nullptr: rows [32*b, +32) of set 1, b grid-strided; otherwise entries [32*b, +32) of the row list (*nrows
// entries).  gate != nullptr: *gate != 0 scans every row, else only the listed ones (the tensor path's fallback).
// part == nullptr: one slice, the results go to idx / score; otherwise slice y writes part[(y * rowsCap + entry)].
__global__ void __launch_bounds__(KX_THREADS)
knn_exact_kernel(const SiftPoint *__restrict__ sift1, const SiftPoint *__restrict__ sift2, int n1, int n2,
                 const int *__restrict__ rows, const unsigned int *__restrict__ nrows, const unsigned int *__restrict__ gate,
                 int2 *__restrict__ idx, float2 *__restrict__ score, Top2 *__restrict__ part, int rowsCap)
{
  if (gate) {
    if (*gate != 0) rows = nullptr;
    else if (!rows) return;
  }
  __shared__ float4 s_a[KX_ROWS * KX_LD];
  __shared__ float4 s_b[KX_COLS * KX_LD];
  const int tid = threadIdx.x;
  const int rq = tid & 15;       // rows rq and rq+16 of the CTA's 32
  const int pt = tid >> 4;       // candidates 4*pt..4*pt+3 of each step
  if (rows) n1 = min((int)*nrows, n1);
  const int nblk = (n2 + KX_COLS - 1) / KX_COLS;
  const int per = (nblk + gridDim.y - 1) / gridDim.y;
  const int b0 = blockIdx.y * per, b1 = min(nblk, b0 + per);
  for (int bp1 = blockIdx.x * KX_ROWS; bp1 < n1; bp1 += gridDim.x * KX_ROWS) {
    __syncthreads();
    for (int i = tid; i < KX_ROWS * 32; i += KX_THREADS) {
      const int r = i >> 5, d = i & 31;
      int p1 = min(bp1 + r, n1 - 1);
      if (rows) p1 = rows[p1];
      s_a[r * KX_LD + d] = reinterpret_cast<const float4 *>(sift1[p1].data)[d];
    }
    Top2 st[2];
    top2_init(st[0]); top2_init(st[1]);
    for (int b = b0; b < b1; b++) {
      __syncthreads();
      for (int i = tid; i < KX_COLS * 32; i += KX_THREADS) {
        const int r = i >> 5, d = i & 31, p2 = b * KX_COLS + r;
        s_b[r * KX_LD + d] = p2 < n2 ? __ldg(reinterpret_cast<const float4 *>(sift2[p2].data) + d)
                                     : make_float4(0.0f, 0.0f, 0.0f, 0.0f);   // zeros score 0: never a neighbour
      }
      __syncthreads();
      float acc[2][4];
#pragma unroll
      for (int i = 0; i < 2; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0.0f;
#pragma unroll 4
      for (int d = 0; d < 32; d++) {
        const float4 a0 = s_a[rq * KX_LD + d], a1 = s_a[(rq + 16) * KX_LD + d];
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const float4 bv = s_b[(4 * pt + j) * KX_LD + d];
          acc[0][j] = __fmaf_rn(a0.x, bv.x, acc[0][j]);
          acc[0][j] = __fmaf_rn(a0.y, bv.y, acc[0][j]);
          acc[0][j] = __fmaf_rn(a0.z, bv.z, acc[0][j]);
          acc[0][j] = __fmaf_rn(a0.w, bv.w, acc[0][j]);
          acc[1][j] = __fmaf_rn(a1.x, bv.x, acc[1][j]);
          acc[1][j] = __fmaf_rn(a1.y, bv.y, acc[1][j]);
          acc[1][j] = __fmaf_rn(a1.z, bv.z, acc[1][j]);
          acc[1][j] = __fmaf_rn(a1.w, bv.w, acc[1][j]);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int p2 = b * KX_COLS + 4 * pt + j;
        top2_insert(st[0], acc[0][j], p2);
        top2_insert(st[1], acc[1][j], p2);
      }
    }
    __syncthreads();
    // publish the (row, thread) states, then one thread per row merges its eight
    Top2 *m = reinterpret_cast<Top2 *>(s_b);
    m[pt * KX_ROWS + rq] = st[0];
    m[pt * KX_ROWS + rq + 16] = st[1];
    __syncthreads();
    const int e = bp1 + tid;
    if (tid < KX_ROWS && e < n1) {
      Top2 t = m[tid];
      for (int y = 1; y < 8; y++) {
        const Top2 o = m[y * KX_ROWS + tid];
        top2_insert(t, o.s1, o.j1);
        top2_insert(t, o.s2, o.j2);
      }
      if (part) {
        part[(size_t)blockIdx.y * rowsCap + e] = t;
      } else {
        const int row = rows ? rows[e] : e;
        idx[row] = make_int2(t.j1, t.j2);
        score[row] = make_float2(t.s1, t.s2);
      }
    }
  }
}

// One thread per entry: the slices' top two, combined.  Same row selection as knn_exact_kernel.
__global__ void __launch_bounds__(256)
knn_merge_kernel(int n1, const int *__restrict__ rows, const unsigned int *__restrict__ nrows,
                 const unsigned int *__restrict__ gate, const Top2 *__restrict__ part, int rowsCap, int slices,
                 int2 *__restrict__ idx, float2 *__restrict__ score)
{
  if (gate) {
    if (*gate != 0) rows = nullptr;
    else if (!rows) return;
  }
  if (rows) n1 = min((int)*nrows, n1);
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n1; e += gridDim.x * blockDim.x) {
    Top2 t = part[e];
    for (int y = 1; y < slices; y++) {
      const Top2 o = part[(size_t)y * rowsCap + e];
      top2_insert(t, o.s1, o.j1);
      top2_insert(t, o.s2, o.j2);
    }
    const int row = rows ? rows[e] : e;
    idx[row] = make_int2(t.j1, t.j2);
    score[row] = make_float2(t.s1, t.s2);
  }
}

// Slices of the candidate range: enough CTAs for two per SM when the rows alone do not provide them, and at least
// KX_MIN_STEPS candidate steps per slice.
static int knn_slices(int rowBlocks, int n2, int sms)
{
  const int steps = idivup(n2, KX_COLS);
  int s = idivup(2 * sms, rowBlocks);
  const int most = idivup(steps, KX_MIN_STEPS);
  if (s > most) s = most;
  if (s > KX_MAX_SLICES) s = KX_MAX_SLICES;
  return s < 1 ? 1 : s;
}

// More than one slice: the slices' partial results go to c.knnPartials.
static int knn_launch(DeviceCtx &c, const SiftPoint *s1, int n1, const SiftPoint *s2, int n2, int *idx, float *score,
                      const int *rows, const unsigned int *nrows, const unsigned int *gate, int rowBlocks, int slices)
{
  int2 *i2 = reinterpret_cast<int2 *>(idx);
  float2 *f2 = reinterpret_cast<float2 *>(score);
  Top2 *part = nullptr;
  if (slices > 1) {
    int r;
    if ((r = c.knnPartials.grow((size_t)slices * n1 * sizeof(Top2))) < 0) return r;
    part = c.knnPartials.as<Top2>();
  }
  knn_exact_kernel<<<dim3(rowBlocks, slices), KX_THREADS, 0, c.stream>>>(s1, s2, n1, n2, rows, nrows, gate, i2, f2, part,
                                                                         n1);
  count_launch();
  if (part) {
    const int blocks = idivup(n1, 256) < 264 ? idivup(n1, 256) : 264;
    knn_merge_kernel<<<blocks, 256, 0, c.stream>>>(n1, rows, nrows, gate, part, n1, slices, i2, f2);
    count_launch();
  }
  CS_CUDA(cudaGetLastError());
  return 0;
}

// Every row of set 1 (mode 1 and small sets).
int knn_exact(DeviceCtx &c, const SiftPoint *s1, int n1, const SiftPoint *s2, int n2, int *idx, float *score)
{
  if (n1 <= 0 || n2 <= 0) return 0;
  const int rowBlocks = idivup(n1, KX_ROWS);
  const int slices = knn_slices(rowBlocks, n2, c.sms);
  return knn_launch(c, s1, n1, s2, n2, idx, score, nullptr, nullptr, nullptr, rowBlocks, slices);
}

// Fallback of a batch wave: the {direction, row} entries its resolve listed (*numEntries, at most cap), each row of its
// own direction's set 1 against all n2 candidates of that direction's set 2.  Rows of one wave belong to different sets,
// so there is no candidate tile to share as in knn_exact_kernel: one warp per entry, the row in shared memory, each lane
// two candidates at a time with their own FMA chains, then the lanes' top two merged by a butterfly (the order is
// total, so the result does not depend on which lane saw which candidate).  Grid-strided: the work is the listed rows
// times their candidates, whatever the number of directions.
#define KL_WARPS 8
__global__ void __launch_bounds__(32 * KL_WARPS)
knn_list_kernel(const MbDir *__restrict__ dirs, const int2 *__restrict__ entries, const unsigned int *__restrict__ numEntries,
                int cap)
{
  __shared__ float4 s_a[KL_WARPS][32];
  const unsigned int FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int n = min((int)*numEntries, cap);
  for (int e = blockIdx.x * KL_WARPS + w; e < n; e += gridDim.x * KL_WARPS) {
    const int2 en = entries[e];
    const MbDir &D = dirs[en.x];
    const SiftPoint *__restrict__ s2 = D.s2;
    const int n2 = D.n2;
    __syncwarp();
    s_a[w][lane] = __ldg(reinterpret_cast<const float4 *>(D.s1[en.y].data) + lane);
    __syncwarp();
    Top2 t;
    top2_init(t);
    for (int j = lane; j < n2; j += 64) {
      const int k = j + 32;
      const float4 *b0 = reinterpret_cast<const float4 *>(s2[j].data);
      const float4 *b1 = reinterpret_cast<const float4 *>(s2[k < n2 ? k : j].data);
      float acc0 = 0.0f, acc1 = 0.0f;       // the reference's score: sequential k = 0..127 FMA chain from 0
#pragma unroll 8
      for (int d = 0; d < 32; d++) {
        const float4 a = s_a[w][d], x = __ldg(b0 + d), y = __ldg(b1 + d);
        acc0 = __fmaf_rn(a.x, x.x, acc0); acc1 = __fmaf_rn(a.x, y.x, acc1);
        acc0 = __fmaf_rn(a.y, x.y, acc0); acc1 = __fmaf_rn(a.y, y.y, acc1);
        acc0 = __fmaf_rn(a.z, x.z, acc0); acc1 = __fmaf_rn(a.z, y.z, acc1);
        acc0 = __fmaf_rn(a.w, x.w, acc0); acc1 = __fmaf_rn(a.w, y.w, acc1);
      }
      top2_insert(t, acc0, j);
      if (k < n2) top2_insert(t, acc1, k);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float t1 = __shfl_xor_sync(FULL, t.s1, o), t2 = __shfl_xor_sync(FULL, t.s2, o);
      const int k1 = __shfl_xor_sync(FULL, t.j1, o), k2 = __shfl_xor_sync(FULL, t.j2, o);
      top2_insert(t, t1, k1);
      top2_insert(t, t2, k2);
    }
    if (lane == 0) {
      D.idx[en.y] = make_int2(t.j1, t.j2);
      D.score[en.y] = make_float2(t.s1, t.s2);
    }
  }
}

int launch_knn_list_fallback(DeviceCtx &c, const MbDir *dirs, const int2 *entries, const unsigned int *numEntries, int cap)
{
  knn_list_kernel<<<4 * c.sms, 32 * KL_WARPS, 0, c.stream>>>(dirs, entries, numEntries, cap);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

// Fallback of the tensor path, decided on the device: the listed rows (usually a few, so the slices are chosen for one
// row block), or every row if *gate != 0 (grid-strided over at most 296 row blocks).
int knn_exact_fallback(DeviceCtx &c, const SiftPoint *s1, int n1, const SiftPoint *s2, int n2, int *idx, float *score,
                       const int *rows, const unsigned int *nrows, const unsigned int *gate)
{
  if (n1 <= 0 || n2 <= 0) return 0;
  const int rowBlocks = idivup(n1, KX_ROWS) < 296 ? idivup(n1, KX_ROWS) : 296;
  return knn_launch(c, s1, n1, s2, n2, idx, score, rows, nrows, gate, rowBlocks, knn_slices(1, n2, c.sms));
}

}  // namespace cs
