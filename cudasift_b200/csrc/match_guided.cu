// match_guided.cu -- guided matching: the two nearest neighbours of every row among the candidates a homography or a
// fundamental matrix admits (cs_match_knn2_guided, cs_match_guided).
//
// Semantics: those of knn_exact (match_knn.cu: the reference's sequential 128-step FMA chain, scores > 0, the order
// (score descending, index ascending)), restricted to the pairs (i, j) with admissible(i, j).  The predicate is the
// FP32 statement of include/cudasift_b200.h: every operation one rounding (__fmul_rn / __fadd_rn / __fsub_rn), set-1
// coefficients {l0, l1, l2, a} (F) or {px, py, pw} (H) and set-2 coefficients {u, v, b}, computed once per point.
// Both directions evaluate the same function on the same operands, so admissibility never depends on the direction.
//
// Every score is exact, so there is nothing to certify: the work is to visit few candidates.  Per direction:
//   1. prep     (both sets, one launch) the coefficient records, the index position of every candidate, the bounding
//               box of those positions, max a over set 1 and max b over set 2.
//   2. index    a cell grid over the box (cell size from the box and the count, on the device), a counting sort of
//               the candidates into it (histogram, scan, scatter) with two sorted copies of the coefficient records:
//               column-major and row-major, so that a cell column or a cell row is one contiguous range.
//   3. knn      one warp per row: the cells the row's admissible region can reach (a disc for H, a strip for F, see
//               DESIGN.md section 4 for the bounds), the predicate on their candidates, the exact chain on the
//               admissible ones (queued so that all 32 lanes run chains together), a butterfly merge of the lanes'
//               top two.  The order is total, so the atomic order inside a cell does not matter.
// A row for which the bounds do not hold (coordinates beyond 1e12, |pw| < 1e-12, an extreme threshold) scans every
// candidate: that is correct, only slower.
//
// Every call runs as waves of jobs (guided_enqueue; a single call is one job): every kernel takes a device table of
// entries in which a CTA finds its own by its index (table_find over CTA bases the host summed).  Each job has its own
// slice of everything, so a row's result depends only on its job: see DESIGN.md section 4.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "ordered_list.cuh"

namespace cs {

#define GD_PER_CELL 2.0       // candidates per cell the grid aims at
#define GD_MAX_SIDE 2048      // cells per grid side at most
#define GD_SLACK 1e-6         // relative slack of the culling bounds (about 16 FP32 roundings)
#define GD_SAFE_POS 1e12f     // the bounds hold for |xpos|, |ypos| up to this
#define GD_SAFE_PW 1e-12f     // ... and, for H, |pw| of set-1 points at least this
#define GD_WARPS 8            // rows per CTA of the knn kernel (one warp each)

// The model as the predicate uses it: entries of the unit-Frobenius model rounded to float, t2 = fl(thresh * thresh).
struct GuidedModel {
  int model;          // CS_GEOM_HOMOGRAPHY or CS_GEOM_FUNDAMENTAL
  float f[9];
  float t2;
};

// One point of either set: its predicate coefficients (NaN when its position is not finite), its position, and its
// index position as a candidate (NaN: not indexed, because it can never be admissible or its direction is not built).
struct GPoint {
  float4 coef;
  float2 pos, key;
};

// Zeroed before every call.  Direction 0: set 1's rows against set 2's candidates; direction 1: the reverse.
struct GHdr {
  unsigned int bb[2][4];        // ordered keys: ~min x, ~min y, max x, max y of the index positions
  unsigned int count[2];        // indexed candidates
  unsigned int maxA, maxB;      // float bits: max a over set 1's indexed points, max b over set 2's
  unsigned int unsafe[2];       // an indexed candidate outside the range where the bounds hold
  unsigned long long stats[4];  // cs_match_guided_stats
};

struct GGrid {
  float x0, y0, x1, y1, inv;    // the box and 1 / cell size
  double cs;                    // 1 / inv
  int gx, gy;
};

// One job as prep, hist, scan and scatter see it: its sets, model and header, its points, cell/slot array, cell counts
// (cap0 / cap1 cells at most per direction), exclusive starts and sorted candidate copies per direction (0: set 2's
// candidates, 1: set 1's, built when dirs == 2).  Job q owns the point CTAs (ceil((n1 + n2) / 256)) from cta0 on and
// the scan CTAs (2 * dirs) from scan0 on.
struct GJob {
  const SiftPoint *s1, *s2;
  int n1, n2, dirs, cap0, cap1;
  GuidedModel gm;
  GHdr *h;
  GPoint *pts;
  int2 *cellSlot;
  unsigned int *counts0, *counts1;
  unsigned int *start0C, *start0R, *start1C, *start1R;
  float4 *coef0C, *coef0R, *coef1C, *coef1R;
  int *idx0C, *idx0R, *idx1C, *idx1R;
  int cta0, scan0;
};

// One direction of a job, as the knn kernel sees it.  The entry owns the CTAs (ceil(nRows / GD_WARPS)) from cta0 on.
struct GDir {
  const SiftPoint *rowSift, *candSift;
  const GPoint *rowPts;
  int nRows, dir, capCells;
  const float4 *coefC, *coefR;  // sorted candidate coefficients, column-major and row-major cell order
  const int *idxC, *idxR;
  const unsigned int *startC, *startR;   // [cells + 1]
  int2 *idx;
  float2 *score;
  GuidedModel gm;
  GHdr *h;                      // the job's header; the statistics are summed into h->stats
  int cull;                     // the threshold allows the culling bounds
  int cta0;
};

// The entry of this CTA and the CTA's index within it (blk): the table's entry whose CTA range (from its `start` field
// on) holds blockIdx.x.
template <class T>
__device__ __forceinline__ T gd_entry(const T *__restrict__ tab, int n, int T::*start, int &blk)
{
  const T e = tab[table_find(tab, n, start, (int)blockIdx.x)];
  blk = (int)blockIdx.x - e.*start;
  return e;
}

// (a0 * x + a1 * y) + a2, three roundings
__device__ __forceinline__ float dot3(float a0, float a1, float a2, float x, float y)
{
  return __fadd_rn(__fadd_rn(__fmul_rn(a0, x), __fmul_rn(a1, y)), a2);
}

// The contract's predicate: c1 = set-1 coefficients, c2 = set-2 coefficients {u, v, b}.
__device__ __forceinline__ bool admissible(int model, float4 c1, float4 c2, float t2)
{
  if (model == CS_GEOM_FUNDAMENTAL) {
    const float num = dot3(c1.x, c1.y, c1.z, c2.x, c2.y);
    return __fmul_rn(num, num) < __fmul_rn(t2, __fadd_rn(c1.w, c2.z));
  }
  const float dx = __fsub_rn(__fmul_rn(c2.x, c1.z), c1.x), dy = __fsub_rn(__fmul_rn(c2.y, c1.z), c1.y);
  return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) < __fmul_rn(t2, __fmul_rn(c1.z, c1.z));
}

// The cell grid of a direction, the same in every thread that asks.  At most max(GD_MAX_SIDE^2, capCells) cells:
// cells beyond the cap merge into the last column / row.
__device__ GGrid grid_of(const GHdr &h, int dir, int capCells)
{
  GGrid g;
  if (h.count[dir] == 0) {
    g.x0 = g.y0 = g.x1 = g.y1 = 0.0f; g.inv = 1.0f; g.cs = 1.0; g.gx = g.gy = 1;
    return g;
  }
  g.x0 = key_float(~h.bb[dir][0]); g.y0 = key_float(~h.bb[dir][1]);
  g.x1 = key_float(h.bb[dir][2]); g.y1 = key_float(h.bb[dir][3]);
  const double n = (double)h.count[dir];
  const double wx = (double)g.x1 - g.x0, wy = (double)g.y1 - g.y0, w = fmax(wx, wy);
  double cs = fmax(sqrt(wx * wy * GD_PER_CELL / n), w * GD_PER_CELL / n);
  cs = fmax(cs, w / (GD_MAX_SIDE - 1));
  if (!(cs > 0.0)) cs = 1.0;                                 // one position (or none)
  g.inv = fmaxf((float)(1.0 / cs), 1e-37f);
  g.cs = 1.0 / (double)g.inv;
  g.gx = (int)fmin(wx / g.cs, GD_MAX_SIDE - 1.0) + 1;
  g.gy = (int)fmin(wy / g.cs, GD_MAX_SIDE - 1.0) + 1;
  while ((long long)g.gx * g.gy > capCells) {
    if (g.gx >= g.gy) g.gx = (g.gx + 1) / 2;
    else g.gy = (g.gy + 1) / 2;
  }
  return g;
}

// The cell coordinate of p: floor((p - p0) * inv) clamped to [0, g).  Monotone in p, which the bounds rely on.
__device__ __forceinline__ int cell_of(float p, float p0, float inv, int g)
{
  return (int)fminf(fmaxf(__fmul_rn(__fsub_rn(p, p0), inv), 0.0f), (float)(g - 1));
}

// ---- 1. prep ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
guided_prep_kernel(const GJob *__restrict__ jobs, int numJobs)
{
  int blk;
  const GJob jb = gd_entry(jobs, numJobs, &GJob::cta0, blk);
  const SiftPoint *__restrict__ s1 = jb.s1, *__restrict__ s2 = jb.s2;
  const int n1 = jb.n1, dirs = jb.dirs;
  const GuidedModel &gm = jb.gm;
  GPoint *__restrict__ pts = jb.pts;
  GHdr *__restrict__ h = jb.h;
  const float *f = gm.f;
  const float nan = __int_as_float(0x7fffffff);
  const int n = n1 + jb.n2, lane = threadIdx.x & 31;
  for (int base = blk * blockDim.x; base < n; base += ((n + 255) >> 8) * blockDim.x) {
    const int t = base + threadIdx.x;
    bool indexed = false, safe = true;
    float maxA = 0.0f, maxB = 0.0f;
    const int dir = t < n1 ? 1 : 0;                          // the direction in which the point is a candidate
    GPoint g;
    g.key = make_float2(nan, nan);
    if (t < n) {
      const SiftPoint &s = dir ? s1[t] : s2[t - n1];
      const float x = s.xpos, y = s.ypos;
      g.pos = make_float2(x, y);
      g.coef = make_float4(nan, nan, nan, nan);
      g.key = make_float2(x, y);
      indexed = isfinite(x) && isfinite(y) && (dir == 0 || dirs == 2);
      safe = fabsf(x) <= GD_SAFE_POS && fabsf(y) <= GD_SAFE_POS;
      if (isfinite(x) && isfinite(y)) {
        if (dir == 1 && gm.model == CS_GEOM_FUNDAMENTAL) {
          const float l0 = dot3(f[0], f[1], f[2], x, y), l1 = dot3(f[3], f[4], f[5], x, y);
          const float l2 = dot3(f[6], f[7], f[8], x, y);
          const float a = __fadd_rn(__fmul_rn(l0, l0), __fmul_rn(l1, l1));
          g.coef = make_float4(l0, l1, l2, a);
          if (indexed && !isnan(a)) maxA = a;
        } else if (dir == 1) {
          const float px = dot3(f[0], f[1], f[2], x, y), py = dot3(f[3], f[4], f[5], x, y);
          const float pw = dot3(f[6], f[7], f[8], x, y);
          g.coef = make_float4(px, py, pw, 0.0f);
          // pw == 0 or a non-finite coefficient admits nothing; the predicted point is the index position
          indexed = indexed && pw != 0.0f && isfinite(px) && isfinite(py) && isfinite(pw);
          safe = safe && fabsf(pw) >= GD_SAFE_PW;
          g.key = make_float2(fminf(fmaxf(__fdiv_rn(px, pw), -FLT_MAX), FLT_MAX),
                              fminf(fmaxf(__fdiv_rn(py, pw), -FLT_MAX), FLT_MAX));
        } else {
          float b = 0.0f;
          if (gm.model == CS_GEOM_FUNDAMENTAL) {
            const float m0 = dot3(f[0], f[3], f[6], x, y), m1 = dot3(f[1], f[4], f[7], x, y);
            b = __fadd_rn(__fmul_rn(m0, m0), __fmul_rn(m1, m1));
            if (indexed && !isnan(b)) maxB = b;
          }
          g.coef = make_float4(x, y, b, 0.0f);
        }
      }
      if (!indexed) g.key = make_float2(nan, nan);
      pts[t] = g;
    }
    // warp-reduced atomics, per direction
    const unsigned int FULL = 0xffffffffu;
    for (int d = 0; d < 2; d++) {
      const bool mine = indexed && dir == d;
      const unsigned int cnt = __reduce_add_sync(FULL, mine ? 1u : 0u);
      const unsigned int k0 = __reduce_max_sync(FULL, mine ? ~float_key(g.key.x) : 0u);
      const unsigned int k1 = __reduce_max_sync(FULL, mine ? ~float_key(g.key.y) : 0u);
      const unsigned int k2 = __reduce_max_sync(FULL, mine ? float_key(g.key.x) : 0u);
      const unsigned int k3 = __reduce_max_sync(FULL, mine ? float_key(g.key.y) : 0u);
      const unsigned int bad = __reduce_or_sync(FULL, (mine && !safe) ? 1u : 0u);
      if (lane == 0 && cnt) {
        atomicAdd(&h->count[d], cnt);
        atomicMax(&h->bb[d][0], k0); atomicMax(&h->bb[d][1], k1);
        atomicMax(&h->bb[d][2], k2); atomicMax(&h->bb[d][3], k3);
        if (bad) atomicOr(&h->unsafe[d], 1u);
      }
    }
    const unsigned int ma = __reduce_max_sync(FULL, __float_as_uint(maxA));   // non-negative floats: bit order
    const unsigned int mb = __reduce_max_sync(FULL, __float_as_uint(maxB));
    if (lane == 0 && ma) atomicMax(&h->maxA, ma);
    if (lane == 0 && mb) atomicMax(&h->maxB, mb);
  }
}

// ---- 2. index -----------------------------------------------------------------------------------------------------
// Per indexed point: its cell (cx * gy + cy) and its slot inside the cell.
__global__ void __launch_bounds__(256)
guided_hist_kernel(const GJob *__restrict__ jobs, int numJobs)
{
  __shared__ GGrid sg[2];
  int blk;
  const GJob jb = gd_entry(jobs, numJobs, &GJob::cta0, blk);
  const GPoint *__restrict__ pts = jb.pts;
  const GHdr *__restrict__ h = jb.h;
  unsigned int *counts0 = jb.counts0, *counts1 = jb.counts1;
  int2 *__restrict__ cellSlot = jb.cellSlot;
  const int n1 = jb.n1, n = n1 + jb.n2;
  if (threadIdx.x < 2) sg[threadIdx.x] = grid_of(*h, threadIdx.x, threadIdx.x ? jb.cap1 : jb.cap0);
  __syncthreads();
  for (int t = blk * blockDim.x + threadIdx.x; t < n; t += ((n + 255) >> 8) * blockDim.x) {
    const float2 k = pts[t].key;
    if (isnan(k.x)) { cellSlot[t] = make_int2(-1, 0); continue; }
    const int d = t < n1 ? 1 : 0;
    const GGrid &g = sg[d];
    const int cell = cell_of(k.x, g.x0, g.inv, g.gx) * g.gy + cell_of(k.y, g.y0, g.inv, g.gy);
    cellSlot[t] = make_int2(cell, (int)atomicAdd((d ? counts1 : counts0) + cell, 1u));
  }
}

// Exclusive scans of the cell counts: CTA 2 * dir + order, order 0 column-major (cell cx * gy + cy), order 1
// row-major (cy * gx + cx).  start[cells] = the count.
__global__ void __launch_bounds__(1024)
guided_scan_kernel(const GJob *__restrict__ jobs, int numJobs)
{
  __shared__ unsigned int s_w[32];
  int blk;
  const GJob jb = gd_entry(jobs, numJobs, &GJob::scan0, blk);
  const int dir = blk >> 1, order = blk & 1;
  const GGrid g = grid_of(*jb.h, dir, dir ? jb.cap1 : jb.cap0);
  const unsigned int *cnt = dir ? jb.counts1 : jb.counts0;
  unsigned int *out = dir ? (order ? jb.start1R : jb.start1C) : (order ? jb.start0R : jb.start0C);
  const int cells = g.gx * g.gy, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned int carry = 0;
  for (int e0 = 0; e0 < cells; e0 += 1024) {
    const int e = e0 + threadIdx.x;
    unsigned int v = 0;
    if (e < cells) v = cnt[order ? (e % g.gx) * g.gy + e / g.gx : e];
    unsigned int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) s_w[w] = inc;
    __syncthreads();
    if (w == 0) {
      const unsigned int c = s_w[lane];
      unsigned int wi = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned int t = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += t;
      }
      s_w[lane] = wi - c;
    }
    __syncthreads();
    if (e < cells) out[e] = carry + s_w[w] + inc - v;
    const unsigned int chunk = __shfl_sync(0xffffffffu, s_w[31] + inc, 31);   // valid in warp 31
    __syncthreads();
    if (threadIdx.x == 1023) s_w[0] = chunk;
    __syncthreads();
    carry += s_w[0];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[cells] = carry;
}

__global__ void __launch_bounds__(256)
guided_scatter_kernel(const GJob *__restrict__ jobs, int numJobs)
{
  __shared__ int sgx[2], sgy[2];
  int blk;
  const GJob jb = gd_entry(jobs, numJobs, &GJob::cta0, blk);
  const GPoint *__restrict__ pts = jb.pts;
  const int2 *__restrict__ cellSlot = jb.cellSlot;
  const int n1 = jb.n1, n = n1 + jb.n2;
  if (threadIdx.x < 2) {
    const GGrid g = grid_of(*jb.h, threadIdx.x, threadIdx.x ? jb.cap1 : jb.cap0);
    sgx[threadIdx.x] = g.gx; sgy[threadIdx.x] = g.gy;
  }
  __syncthreads();
  for (int t = blk * blockDim.x + threadIdx.x; t < n; t += ((n + 255) >> 8) * blockDim.x) {
    const int2 cl = cellSlot[t];
    if (cl.x < 0) continue;
    const int d = t < n1 ? 1 : 0, gx = sgx[d], gy = sgy[d];
    const int cx = cl.x / gy, cy = cl.x - cx * gy;
    const unsigned int pc = (d ? jb.start1C : jb.start0C)[cl.x] + cl.y;
    const unsigned int pr = (d ? jb.start1R : jb.start0R)[cy * gx + cx] + cl.y;
    const float4 c = pts[t].coef;
    const int i = d ? t : t - n1;
    (d ? jb.coef1C : jb.coef0C)[pc] = c; (d ? jb.idx1C : jb.idx0C)[pc] = i;
    (d ? jb.coef1R : jb.coef0R)[pr] = c; (d ? jb.idx1R : jb.idx0R)[pr] = i;
  }
}

// ---- 3. knn -------------------------------------------------------------------------------------------------------
// The reference's score: the sequential k = 0..127 FMA chain from 0, as knn_exact_kernel computes it.
__device__ __forceinline__ float chain_score(const float4 *a, const float4 *__restrict__ b)
{
  float acc = 0.0f;
#pragma unroll 8
  for (int d = 0; d < 32; d++) {
    const float4 av = a[d], bv = __ldg(b + d);
    acc = __fmaf_rn(av.x, bv.x, acc);
    acc = __fmaf_rn(av.y, bv.y, acc);
    acc = __fmaf_rn(av.z, bv.z, acc);
    acc = __fmaf_rn(av.w, bv.w, acc);
  }
  return acc;
}

// What a row visits: nothing, every candidate, the cell box [c0, c1] x [r0, r1] (H), or the strip
// |L0 X + L1 Y + L2| <= W (F) walked by cell columns (|L1| >= |L0|) or by cell rows.
enum { GK_NONE, GK_ALL, GK_BOX, GK_COLS, GK_ROWS };
struct Region {
  int kind, c0, c1, r0, r1;
  double L0, L1, L2, W;
};

__device__ __forceinline__ double fabs_max(float a, float b) { return fmax(fabs((double)a), fabs((double)b)); }

__device__ Region row_region(const GDir &d, const GPoint &rp, const GuidedModel &gm, const GGrid &g, double kmax,
                             bool cull)
{
  Region R;
  R.kind = GK_ALL;
  const float *f = gm.f;
  const double E = GD_SLACK, x = rp.pos.x, y = rp.pos.y;
  const double ucand = fabs_max(g.x0, g.x1) + fabs_max(g.y0, g.y1);   // |X| + |Y| of every candidate, at most
  bool safe = cull && fabs(x) <= GD_SAFE_POS && fabs(y) <= GD_SAFE_POS;
  if (gm.model == CS_GEOM_HOMOGRAPHY) {
    double cx = x, cy = y;
    if (d.dir == 0) {
      const float px = rp.coef.x, py = rp.coef.y, pw = rp.coef.z;
      if (!(pw != 0.0f && isfinite(px) && isfinite(py) && isfinite(pw))) { R.kind = GK_NONE; return R; }
      safe = safe && fabsf(pw) >= GD_SAFE_PW;
      cx = (double)px / pw; cy = (double)py / pw;
    }
    if (!safe) return R;
    const double rad = sqrt((double)gm.t2) * (1.0 + E) + E * (1.0 + fabs(cx) + fabs(cy) + ucand);
    const double xl = cx - rad, xh = cx + rad, yl = cy - rad, yh = cy + rad;
    if (!(isfinite(xl) && isfinite(xh) && isfinite(yl) && isfinite(yh))) return R;
    if (xh < g.x0 || xl > g.x1 || yh < g.y0 || yl > g.y1) { R.kind = GK_NONE; return R; }
    R.kind = GK_BOX;
    R.c0 = cell_of(__double2float_rd(xl), g.x0, g.inv, g.gx); R.c1 = cell_of(__double2float_ru(xh), g.x0, g.inv, g.gx);
    R.r0 = cell_of(__double2float_rd(yl), g.y0, g.inv, g.gy); R.r1 = cell_of(__double2float_ru(yh), g.y0, g.inv, g.gy);
    return R;
  }
  if (!safe) return R;
  // The row's line in the candidates' image, in double: F x1 (direction 0) or F^T x2 (direction 1).  The FP32 num
  // differs from x2^T F x1 by at most about 6 roundings of |x2|^T |F| |x1|; g bounds that row's |F| |x1| or
  // |F|^T |x2|, and the candidates' |X|, |Y| are at most those of the box.
  double own, g0, g1, g2;                                     // own: the row's a (direction 0) or b (direction 1)
  const int s = d.dir == 0 ? 1 : 3, o = d.dir == 0 ? 3 : 1;   // strides of f along and across the line's entries
  R.L0 = (double)f[0] * x + (double)f[s] * y + f[2 * s];
  R.L1 = (double)f[o] * x + (double)f[o + s] * y + f[o + 2 * s];
  R.L2 = (double)f[2 * o] * x + (double)f[2 * o + s] * y + f[2 * o + 2 * s];
  g0 = fabs((double)f[0] * x) + fabs((double)f[s] * y) + fabs((double)f[2 * s]);
  g1 = fabs((double)f[o] * x) + fabs((double)f[o + s] * y) + fabs((double)f[o + 2 * s]);
  g2 = fabs((double)f[2 * o] * x) + fabs((double)f[2 * o + s] * y) + fabs((double)f[2 * o + 2 * s]);
  own = d.dir == 0 ? rp.coef.w : rp.coef.z;
  const double slack = E * (g0 * fabs_max(g.x0, g.x1) + g1 * fabs_max(g.y0, g.y1) + g2) + 1e-30;
  R.W = sqrt((double)gm.t2 * (own + kmax)) * (1.0 + E) + slack;
  if (!(isfinite(R.W) && fmax(fabs(R.L0), fabs(R.L1)) > 0.0)) return R;
  R.kind = fabs(R.L1) >= fabs(R.L0) ? GK_COLS : GK_ROWS;
  return R;
}

// Cell line k of a strip (a column for GK_COLS, a row for GK_ROWS): the cells [lo, hi] across it that the strip
// can reach, or false.  a0 / a1 / n: the line's axis; b0 / b1 / m: the other axis.  A candidate in line k has its
// coordinate along the axis in [ua, ub] (the slack covers the rounding of cell_of).
__device__ __forceinline__ bool strip_cells(int k, int n, float a0, float a1, float b0, float b1, int m, double cs,
                                            float inv, double P, double Q, double R2, double W, int &lo, int &hi)
{
  // the strip: |P * s + Q * o + R2| <= W, s along the axis, o across it, |Q| >= |P|
  const double dl = GD_SLACK * (1.0 + fabs((double)a0) + (k + 1) * cs);
  const double ua = k == 0 ? (double)a0 : fmax((double)a0 + k * cs - dl, (double)a0);
  const double ub = k == n - 1 ? (double)a1 : fmin((double)a0 + (k + 1) * cs + dl, (double)a1);
  if (ua > ub) return false;
  const double va = -(P * ua + R2) / Q, vb = -(P * ub + R2) / Q, wv = W / fabs(Q);
  double vl = fmin(va, vb) - wv, vh = fmax(va, vb) + wv;
  vl -= 1e-9 * (1.0 + fabs(vl));
  vh += 1e-9 * (1.0 + fabs(vh));
  if (!(vh >= b0 && vl <= b1)) return false;
  lo = cell_of(__double2float_rd(vl), b0, inv, m);
  hi = cell_of(__double2float_ru(vh), b0, inv, m);
  return true;
}

// Every direction of the table has one CTA per GD_WARPS rows.  d is the table's entry in global memory, read in place:
// a copy would index gm.f from local memory.
__global__ void __launch_bounds__(GD_WARPS * 32)
guided_knn_kernel(const GDir *__restrict__ dirs, int numDirs)
{
  const GDir &d = dirs[table_find(dirs, numDirs, &GDir::cta0, (int)blockIdx.x)];
  const int blk = (int)blockIdx.x - d.cta0, ctas = (d.nRows + GD_WARPS - 1) / GD_WARPS;
  __shared__ float4 s_row[GD_WARPS][32];
  __shared__ int s_q[GD_WARPS][64];
  const GuidedModel &gm = d.gm;
  const GHdr *__restrict__ h = d.h;
  const unsigned int FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const GGrid g = grid_of(*h, d.dir, d.capCells);
  const unsigned int nc = h->count[d.dir];
  const bool cull = d.cull && !h->unsafe[d.dir];
  const double kmax = __uint_as_float(d.dir == 0 ? h->maxB : h->maxA);
  unsigned long long evals = 0, hits = 0, rowsHit = 0;
  for (int r = blk * GD_WARPS + w; r < d.nRows; r += ctas * GD_WARPS) {
    const GPoint rp = d.rowPts[r];
    Top2 t;
    top2_init(t);
    unsigned int rowHits = 0;
    Region R;
    R.kind = GK_NONE;
    if (nc > 0 && isfinite(rp.pos.x) && isfinite(rp.pos.y)) R = row_region(d, rp, gm, g, kmax, cull);
    if (R.kind != GK_NONE) {
      s_row[w][lane] = reinterpret_cast<const float4 *>(d.rowSift[r].data)[lane];
      __syncwarp();
      const bool rowOrder = R.kind == GK_ROWS;
      const float4 *coef = rowOrder ? d.coefR : d.coefC;
      const int *cidx = rowOrder ? d.idxR : d.idxC;
      const int lines = R.kind == GK_ALL ? 1 : R.kind == GK_BOX ? R.c1 - R.c0 + 1 : R.kind == GK_COLS ? g.gx : g.gy;
      int qn = 0;
      for (int base = 0; base < lines; base += 32) {
        // this lane's line: a contiguous range [s, s + len) of the sorted candidates
        const int k = base + lane;
        unsigned int s = 0, len = 0;
        if (k < lines) {
          int lo = 0, hi = -1, line = k, across = 0;
          if (R.kind == GK_ALL) { s = 0; len = nc; }
          else if (R.kind == GK_BOX) { line = R.c0 + k; lo = R.r0; hi = R.r1; across = g.gy; }
          else if (R.kind == GK_COLS) {
            if (!strip_cells(k, g.gx, g.x0, g.x1, g.y0, g.y1, g.gy, g.cs, g.inv, R.L0, R.L1, R.L2, R.W, lo, hi)) hi = -1;
            across = g.gy;
          } else {
            if (!strip_cells(k, g.gy, g.y0, g.y1, g.x0, g.x1, g.gx, g.cs, g.inv, R.L1, R.L0, R.L2, R.W, lo, hi)) hi = -1;
            across = g.gx;
          }
          if (R.kind != GK_ALL && hi >= lo) {
            const unsigned int *st = rowOrder ? d.startR : d.startC;
            s = st[line * across + lo];
            len = st[line * across + hi + 1] - s;
          }
        }
        unsigned int inc = len;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned int v = __shfl_up_sync(FULL, inc, o);
          if (lane >= o) inc += v;
        }
        const unsigned int excl = inc - len, total = __shfl_sync(FULL, inc, 31);
        evals += total;
        for (unsigned int k0 = 0; k0 < total; k0 += 32) {
          const unsigned int e = k0 + lane;
          int src = 0;                                           // the lane whose range holds e
#pragma unroll
          for (int step = 16; step > 0; step >>= 1)
            if (__shfl_sync(FULL, excl, src + step) <= e) src += step;
          const unsigned int p = __shfl_sync(FULL, s, src) + (e - __shfl_sync(FULL, excl, src));
          bool ok = false;
          int j = -1;
          if (e < total) {
            const float4 cc = coef[p];
            ok = d.dir == 0 ? admissible(gm.model, rp.coef, cc, gm.t2) : admissible(gm.model, cc, rp.coef, gm.t2);
            j = cidx[p];
          }
          const unsigned int bal = __ballot_sync(FULL, ok);
          if (ok) s_q[w][qn + __popc(bal & ((1u << lane) - 1u))] = j;
          qn += __popc(bal);
          rowHits += __popc(bal);
          __syncwarp();
          if (qn >= 32) {                                        // every lane runs one chain
            const int jj = s_q[w][lane];
            top2_insert(t, chain_score(s_row[w], reinterpret_cast<const float4 *>(d.candSift[jj].data)), jj);
            __syncwarp();
            if (lane < qn - 32) s_q[w][lane] = s_q[w][lane + 32];
            qn -= 32;
            __syncwarp();
          }
        }
      }
      if (lane < qn) {
        const int jj = s_q[w][lane];
        top2_insert(t, chain_score(s_row[w], reinterpret_cast<const float4 *>(d.candSift[jj].data)), jj);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {                         // butterfly: disjoint halves at every step
        Top2 u;
        u.s1 = __shfl_xor_sync(FULL, t.s1, o); u.j1 = __shfl_xor_sync(FULL, t.j1, o);
        u.s2 = __shfl_xor_sync(FULL, t.s2, o); u.j2 = __shfl_xor_sync(FULL, t.j2, o);
        top2_insert(t, u.s1, u.j1);
        top2_insert(t, u.s2, u.j2);
      }
      __syncwarp();                                              // s_row and s_q are reused by the next row
    }
    hits += rowHits;
    rowsHit += rowHits > 0;
    if (lane == 0) {
      d.idx[r] = make_int2(t.j1, t.j2);
      d.score[r] = make_float2(t.s1, t.s2);
    }
  }
  if (lane == 0 && (evals || rowsHit)) {
    atomicAdd(&d.h->stats[0], evals);
    atomicAdd(&d.h->stats[1], hits);
    atomicAdd(&d.h->stats[2 + d.dir], rowsHit);
  }
}

// ---- host -----------------------------------------------------------------------------------------------------------
static GuidedModel guided_model(int model, const double in[9], float thresh)
{
  GuidedModel gm;
  gm.model = model;
  double s = 0.0;
  for (int k = 0; k < 9; k++) s += in[k] * in[k];
  s = std::sqrt(s);
  for (int k = 0; k < 9; k++) gm.f[k] = (float)(in[k] / s);
  gm.t2 = thresh * thresh;
  return gm;
}

// The scratch of one job (its header aside), every piece 256-byte aligned: the cell counts, zeroed before the wave
// (offsets from the zeroed base), then the rest, its knn lists and pair scratch included (offsets from the other base).
struct GLayout {
  int cap0, cap1;
  size_t cnt0, cnt1, zeroBytes;
  size_t pts, cell, s0C, s0R, s1C, s1R, c0C, i0C, c0R, i0R, c1C, i1C, c1R, i1R;
  size_t idx1, sc1, idx2, sc2, masks, ctaCounts, bytes;
};
static GLayout gd_layout(int n1, int n2, int dirs)
{
  GLayout L;
  const size_t n = (size_t)n1 + n2, m1 = dirs == 2 ? n1 : 1;
  L.cap0 = 2 * n2 + 64;
  L.cap1 = dirs == 2 ? 2 * n1 + 64 : 1;
  Layout z(256), b(256);
  L.cnt0 = z.take(4 * (size_t)L.cap0); L.cnt1 = z.take(4 * (size_t)L.cap1);
  L.zeroBytes = z.bytes;
  L.pts = b.take(sizeof(GPoint) * n); L.cell = b.take(sizeof(int2) * n);
  L.s0C = b.take(4 * ((size_t)L.cap0 + 1)); L.s0R = b.take(4 * ((size_t)L.cap0 + 1));
  L.s1C = b.take(4 * ((size_t)L.cap1 + 1)); L.s1R = b.take(4 * ((size_t)L.cap1 + 1));
  L.c0C = b.take(16 * (size_t)n2); L.i0C = b.take(4 * (size_t)n2);
  L.c0R = b.take(16 * (size_t)n2); L.i0R = b.take(4 * (size_t)n2);
  L.c1C = b.take(16 * m1); L.i1C = b.take(4 * m1); L.c1R = b.take(16 * m1); L.i1R = b.take(4 * m1);
  const size_t l2 = dirs == 2 ? (size_t)n2 : 0;
  L.idx1 = b.take(8 * (size_t)n1); L.sc1 = b.take(8 * (size_t)n1);
  L.idx2 = b.take(8 * l2); L.sc2 = b.take(8 * l2);
  // the pair list's ballot words and CTA counts (ordered_list.cuh)
  L.masks = b.take(4 * (size_t)list_words(n1)); L.ctaCounts = b.take(4 * (size_t)list_ctas(n1));
  L.bytes = b.bytes;
  return L;
}

// The entry of a job: header h, cell counts from z, the rest from b.
static GJob gd_job(const SiftPoint *s1, int n1, const SiftPoint *s2, int n2, int dirs, const GuidedModel &gm, GHdr *h,
                   char *z, char *b, const GLayout &L)
{
  GJob j = {};
  j.s1 = s1; j.n1 = n1; j.s2 = s2; j.n2 = n2; j.dirs = dirs; j.cap0 = L.cap0; j.cap1 = L.cap1;
  j.gm = gm; j.h = h;
  j.counts0 = reinterpret_cast<unsigned int *>(z + L.cnt0); j.counts1 = reinterpret_cast<unsigned int *>(z + L.cnt1);
  auto u32 = [&](size_t o) { return reinterpret_cast<unsigned int *>(b + o); };
  auto f4 = [&](size_t o) { return reinterpret_cast<float4 *>(b + o); };
  auto i32 = [&](size_t o) { return reinterpret_cast<int *>(b + o); };
  j.pts = reinterpret_cast<GPoint *>(b + L.pts); j.cellSlot = reinterpret_cast<int2 *>(b + L.cell);
  j.start0C = u32(L.s0C); j.start0R = u32(L.s0R); j.start1C = u32(L.s1C); j.start1R = u32(L.s1R);
  j.coef0C = f4(L.c0C); j.idx0C = i32(L.i0C); j.coef0R = f4(L.c0R); j.idx0R = i32(L.i0R);
  j.coef1C = f4(L.c1C); j.idx1C = i32(L.i1C); j.coef1R = f4(L.c1R); j.idx1R = i32(L.i1R);
  return j;
}

// Direction dir of a job (0: set 1's rows against set 2, 1: the reverse), its lists at idx / score.
static GDir gd_dir(const GJob &j, int dir, int2 *idx, float2 *score, int cta0)
{
  GDir d;
  d.dir = dir;
  d.rowSift = dir ? j.s2 : j.s1;
  d.candSift = dir ? j.s1 : j.s2;
  d.rowPts = dir ? j.pts + j.n1 : j.pts;
  d.nRows = dir ? j.n2 : j.n1;
  d.capCells = dir ? j.cap1 : j.cap0;
  d.coefC = dir ? j.coef1C : j.coef0C; d.idxC = dir ? j.idx1C : j.idx0C;
  d.coefR = dir ? j.coef1R : j.coef0R; d.idxR = dir ? j.idx1R : j.idx0R;
  d.startC = dir ? j.start1C : j.start0C; d.startR = dir ? j.start1R : j.start0R;
  d.idx = idx; d.score = score;
  d.gm = j.gm; d.h = j.h;
  // the bounds of DESIGN.md section 4 hold for thresholds whose square is a normal float well inside the range
  d.cull = j.gm.t2 >= 1e-6f && j.gm.t2 <= 1e12f;
  d.cta0 = cta0;
  return d;
}

// A job's wave scratch: its layout and GD_JOB_STATE_BYTES for its header and pair total (the header states the rule).
#define GD_JOB_STATE_BYTES 256

// A wave (the header states the rule): the non-empty jobs ne[q0, q1) and what its launches need.
struct GdWave {
  int q0 = 0, q1 = 0, pointCtas = 0, knnCtas = 0, pairCtas = 0, dirs = 0;
  size_t bytes = 0, zeroBytes = 0, restBytes = 0;
  // The tables (jobs at 0, directions at dirsAt, pair jobs at pairJobsAt) and the state (headers at 0, pair totals at
  // totalsAt), each piece at a multiple of 16 bytes.  Pinned (c.h_guidedBatch from pinOff): the tables, then from
  // tabBytes the copied-back state.  Device scratch (c.guided), every piece at a multiple of 256 bytes: the tables;
  // from stateDev, zeroed per wave, the state and every job's cell counts (from zeroDev); from restDev the rest of
  // every job.
  size_t dirsAt = 0, pairJobsAt = 0, tabBytes = 0, totalsAt = 0, stateBytes = 0, pinOff = 0;
  size_t stateDev = 0, zeroDev = 0, restDev = 0;
};

int guided_enqueue(DeviceCtx &c, const cs_match_set *sets, const cs_match_job *jobs, int numJobs, const int *models,
                   const double *models_in, float thresh, float maxRatio, float maxDistance, bool cross,
                   GuidedBatchOut *out, const GuidedSingle *single)
{
  const int D = cross ? 2 : 1;
  const bool knnOnly = single && single->idx;
  std::vector<int> ne;
  for (int p = 0; p < numJobs; p++)
    if (sets[jobs[p].set1].n > 0 && sets[jobs[p].set2].n > 0) ne.push_back(p);
  if (ne.empty()) return 0;
  std::vector<GdWave> waves;
  size_t dev = 0, pin = 0;
  for (int q = 0; q < (int)ne.size(); q++) {
    const cs_match_job &jb = jobs[ne[q]];
    const int n1 = sets[jb.set1].n, n2 = sets[jb.set2].n;
    const GLayout L = gd_layout(n1, n2, D);
    const size_t cost = L.zeroBytes + L.bytes + GD_JOB_STATE_BYTES;
    if (waves.empty() || waves.back().bytes + cost > WAVE_BYTES) {
      waves.emplace_back();
      waves.back().q0 = q;
    }
    GdWave &v = waves.back();
    v.q1 = q + 1;
    v.bytes += cost;
    v.zeroBytes += L.zeroBytes;
    v.restBytes += L.bytes;
    v.pointCtas += idivup(n1 + n2, 256);
    v.knnCtas += idivup(n1, GD_WARPS) + (cross ? idivup(n2, GD_WARPS) : 0);
    v.pairCtas += list_ctas(n1);
  }
  for (GdWave &v : waves) {
    const size_t J = v.q1 - v.q0;
    v.dirs = (int)J * D;
    Layout tab(16), state(16), scratch(256);
    tab.take(J * sizeof(GJob));
    v.dirsAt = tab.take(v.dirs * sizeof(GDir));
    v.pairJobsAt = tab.take(J * sizeof(PairJob));
    v.tabBytes = tab.bytes;
    state.take(J * sizeof(GHdr));
    v.totalsAt = state.take(J * sizeof(unsigned int));
    v.stateBytes = state.bytes;
    v.pinOff = pin;
    pin += v.tabBytes + v.stateBytes;
    scratch.take(v.tabBytes);
    v.stateDev = scratch.take(v.stateBytes);
    v.zeroDev = scratch.take(v.zeroBytes);
    v.restDev = scratch.take(v.restBytes);
    dev = std::max(dev, scratch.bytes);
  }
  int r;
  if ((r = c.guided.grow(dev)) < 0) return r;
  if ((r = c.h_guidedBatch.grow(pin)) < 0) return r;
  const cudaStream_t st = c.stream;
  cudaEvent_t *tev = match_timing_events();
  for (const GdWave &v : waves) {
    const int J = v.q1 - v.q0;
    char *hp = c.h_guidedBatch.as<char>() + v.pinOff;
    GJob *hj = reinterpret_cast<GJob *>(hp);
    GDir *hd = reinterpret_cast<GDir *>(hp + v.dirsAt);
    PairJob *hpj = reinterpret_cast<PairJob *>(hp + v.pairJobsAt);
    const char *hstate = hp + v.tabBytes;
    char *dt = c.guided.as<char>(), *ds = dt + v.stateDev;
    GHdr *hdrs = reinterpret_cast<GHdr *>(ds);
    unsigned int *totals = reinterpret_cast<unsigned int *>(ds + v.totalsAt);
    char *z = dt + v.zeroDev, *b = dt + v.restDev;
    int pointCta = 0, knnCta = 0, pairCta = 0;
    for (int k = 0; k < J; k++) {
      const int p = ne[v.q0 + k];
      const cs_match_job &jb = jobs[p];
      const int n1 = sets[jb.set1].n, n2 = sets[jb.set2].n;
      const GLayout L = gd_layout(n1, n2, D);
      GJob &j = hj[k];
      j = gd_job(static_cast<const SiftPoint *>(sets[jb.set1].pts), n1, static_cast<const SiftPoint *>(sets[jb.set2].pts),
                 n2, D, guided_model(models[p], models_in + 9 * (size_t)p, thresh), hdrs + k, z, b, L);
      j.cta0 = pointCta; j.scan0 = 2 * D * k;
      pointCta += idivup(n1 + n2, 256);
      int2 *idx1 = knnOnly ? reinterpret_cast<int2 *>(single->idx) : reinterpret_cast<int2 *>(b + L.idx1);
      float2 *sc1 = knnOnly ? reinterpret_cast<float2 *>(single->score) : reinterpret_cast<float2 *>(b + L.sc1);
      int2 *idx2 = cross ? reinterpret_cast<int2 *>(b + L.idx2) : nullptr;
      float2 *sc2 = cross ? reinterpret_cast<float2 *>(b + L.sc2) : nullptr;
      for (int dir = 0; dir < D; dir++) {
        hd[D * k + dir] = gd_dir(j, dir, dir ? idx2 : idx1, dir ? sc2 : sc1, knnCta);
        knnCta += idivup(dir ? n2 : n1, GD_WARPS);
      }
      PairJob &pj = hpj[k];
      pj = PairJob{};
      pj.jv = reinterpret_cast<const int *>(idx1); pj.jstride = 2;
      pj.n1 = n1; pj.n2 = n2;
      pj.idx1 = idx1; pj.score1 = sc1; pj.idx2 = idx2; pj.score2 = sc2;
      pj.masks = reinterpret_cast<unsigned int *>(b + L.masks);
      pj.blockCounts = reinterpret_cast<unsigned int *>(b + L.ctaCounts);
      pj.pairs = reinterpret_cast<int2 *>(jb.pairs); pj.maxPairs = jb.maxPairs;
      pj.total = totals + k;
      pj.cta0 = pairCta;
      pairCta += list_ctas(n1);
      out[p].stats = reinterpret_cast<const GHdr *>(hstate)[k].stats;
      out[p].total = reinterpret_cast<const unsigned int *>(hstate + v.totalsAt) + k;
      z += L.zeroBytes;
      b += L.bytes;
    }
    const GJob *dj = reinterpret_cast<const GJob *>(dt);
    const GDir *dd = reinterpret_cast<const GDir *>(dt + v.dirsAt);
    const PairJob *dpj = reinterpret_cast<const PairJob *>(dt + v.pairJobsAt);
    CS_CUDA(cudaMemsetAsync(ds, 0, v.restDev - v.stateDev, st));
    CS_CUDA(cudaMemcpyAsync(dt, hp, v.tabBytes, cudaMemcpyHostToDevice, st));
    if (tev) cudaEventRecord(tev[0], st);
    guided_prep_kernel<<<v.pointCtas, 256, 0, st>>>(dj, J);
    if (tev) cudaEventRecord(tev[1], st);
    guided_hist_kernel<<<v.pointCtas, 256, 0, st>>>(dj, J);
    guided_scan_kernel<<<2 * D * J, 1024, 0, st>>>(dj, J);
    guided_scatter_kernel<<<v.pointCtas, 256, 0, st>>>(dj, J);
    if (tev) cudaEventRecord(tev[2], st);
    guided_knn_kernel<<<v.knnCtas, GD_WARPS * 32, 0, st>>>(dd, v.dirs);
    if (tev) cudaEventRecord(tev[3], st);
    count_launch(5);
    CS_CUDA(cudaGetLastError());
    if (!knnOnly) {
      if ((r = launch_ratio_pairs_batch(c, dpj, J, v.pairCtas, maxRatio, maxDistance)) < 0) return r;
      if (tev) cudaEventRecord(tev[4], st);
    }
    CS_CUDA(cudaMemcpyAsync(hp + v.tabBytes, ds, v.stateBytes, cudaMemcpyDeviceToHost, st));
    static const char *const stages[] = {"prep", "index", "knn", "pairs"};
    if (tev && single)
      report_stage_times(tev, stages, knnOnly ? 3 : 4, "guided timing %dx%d", hj[0].n1, hj[0].n2);
    else if (tev)
      report_stage_times(tev, stages, 4, "guided-batch timing %d jobs %d directions %d rows", J, v.dirs, 8 * v.knnCtas);
  }
  return 0;
}

}  // namespace cs
