// seams.cu -- global seam levelling of a textured mesh (cs_level_texture_seams) after Lempitsky & Ivanov 2007 as
// Waechter, Moehrle & Goesele 2014 apply it: one offset per (vertex, label) pair, seam rows that pull the two sides of
// every seam vertex together and smoothness rows along the edges of each label, their weighted graph Laplacian solved
// by Jacobi-preconditioned CG in one cooperative kernel, and the offsets added to the atlas texel by texel.  Every
// rule is stated in cudasift_b200.h at cs_level_texture_seams; tests/seam_oracle.py restates them in float64.  The edge
// keys, the adjacency and the lower-vertex edge rule are texturing's (trimesh.cuh); the sorted
// incidences, the per-unknown pieces and the three-level totals are coop.cuh's.
//
// Determinism: no floating-point atomics.  Integer atomics only where the result does not depend on their order (the
// input flag, the 64-bit (distance, face) texel keys, the count of visited texels).  Every floating-point sum has a
// fixed order: a seam row's samples in k order per edge, then its edges in sorted key order; an unknown's incidences
// in sorted (row, side) order by coop.cuh's pieces; the totals in coop.cuh's three-level order.  This unit is compiled
// with -fmad=false so that every float64 product and sum is rounded once, in the order written, as the oracle
// computes it.
#include <cassert>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include <cooperative_groups.h>
#include <cub/cub.cuh>

#include "common.cuh"
#include "coop.cuh"
#include "trimesh.cuh"

namespace cg = cooperative_groups;

namespace cs {

namespace {

constexpr unsigned long long NONE = ~0ull;
constexpr int SL_PV = 2;                       // an unknown's piece: the sum of w, then b or the neighbours' w p

// The device words of a call; the host reads them after the input check, the counts and the solve.
struct SeamsResult {
  unsigned int bad, seen;
  int unknowns, seamEdges, smoothRows, seamRows;  // copied from the last entries of their scans
  int iters, converged;
  unsigned long long texels;
  double info[3];
};

// An unknown's sorted incidences [start, end) (coop.cuh's item).
struct SeamUnk {
  int start, end;
};

struct SeamsParams {
  SeamsResult *res;
  int V, T;
  const float *vin;
  const int *tin, *view;
  const float *uv, *atlas;
  float *out, *corner;
  int rows, width, padding, copyAll;
  const int *ctab;                            // [C][8] the chart table
  const int *rowStart, *rowList;              // per atlas row, the charts that cover it by ox
  int *faceChart;                             // [T]
  unsigned long long *ekey, *ekeyS, *ukey, *ukeyS, *skeyS;
  int *eval, *evalS, *uval, *uvalS, *nbr;
  int *uHead, *uScan, *seFlag, *seScan, *sHead, *sScan, *cornerUnk;
  unsigned long long *xkey, *xkeyS;           // [2E] seam ends: (g(v, a) << 32) | g(v, b)
  int *xval, *xvalS, *xHead, *xScan;
  double *xsum;                               // [2E][3]: sum w I_a, sum w I_b, sum w
  int *ri, *rj;                               // [R] rows: g_i - g_j = d with weight w
  double *rw, *rd, *rfa, *rfb;                // rfa, rfb: F_a, F_b of the seam rows
  int *ikey, *ikeyS, *ival, *ivalS;           // [2R] incidences (unknown; 2 row + side)
  SeamUnk *unk;
  double *x, *r, *z, *p, *q, *diag, *b;
  double *pieces, *partA, *groupA, *partB, *groupB, *partE, *groupE;
  unsigned long long *tkey;                   // [rows][width] texel keys
  double smooth, reg, tol2;
  int maxIt, N, E, Rs, Rm;
};

// ---- input (rule 1) -----------------------------------------------------------------------------------------------
// A seen face's chart: the chart of the row index whose rectangle holds floor of corner 0's uv, with the face's label.
__global__ void __launch_bounds__(MT) seams_check_kernel(SeamsParams p)
{
  bool bad = false;
  unsigned int seen = 0;
  for (int f = blockIdx.x * MT + threadIdx.x; f < p.T; f += gridDim.x * MT) {
    const int l = p.view[f];
    int ch = -1;
    if (l >= 0) {
      const float *u = p.uv + 6 * (size_t)f;
      bool fin = true;
      for (int k = 0; k < 6; k++) fin = fin && isfinite(u[k]);
      const double fx = fin ? floor((double)u[0]) : -1.0, fy = fin ? floor((double)u[1]) : -1.0;
      if (fx >= 0.0 && fx < (double)p.width && fy >= 0.0 && fy < (double)p.rows) {
        const int x = (int)fx, y = (int)fy;
        int lo = p.rowStart[y], hi = p.rowStart[y + 1] - 1;   // the last entry with ox <= x
        int at = -1;
        while (lo <= hi) {
          const int mid = (lo + hi) >> 1;
          if (p.ctab[8 * (size_t)p.rowList[mid] + 5] <= x) { at = mid; lo = mid + 1; } else hi = mid - 1;
        }
        if (at >= 0) {
          const int c = p.rowList[at];
          const int *e = p.ctab + 8 * (size_t)c;
          if (x < e[5] + e[3] && e[0] == l) ch = c;
        }
      }
      bad = bad || ch < 0;
      seen++;
    }
    p.faceChart[f] = ch;
  }
  if (bad) atomicOr(&p.res->bad, 1u);
  if (seen) atomicAdd(&p.res->seen, seen);
}

// ---- unknowns, adjacency, smoothness rows and seam edges (rules 2-4) ----------------------------------------------
__global__ void __launch_bounds__(MT) seams_keys_kernel(SeamsParams p)
{
  for (int c = blockIdx.x * MT + threadIdx.x; c < 3 * p.T; c += gridDim.x * MT) {
    p.ekey[c] = edge_key_of(p.tin, c);
    p.eval[c] = c;
    p.nbr[c] = -1;
    const int l = p.view[c / 3];
    p.ukey[c] = l >= 0 ? ((unsigned long long)(unsigned int)p.tin[c] << 32) | (unsigned int)l : NONE;
    p.uval[c] = c;
  }
}

// texturing's adjacency; the first corner of every distinct (vertex, label) key
__global__ void __launch_bounds__(MT) seams_adjacency_kernel(SeamsParams p)
{
  const int n = 3 * p.T;
  for (int i = blockIdx.x * MT + threadIdx.x; i < n; i += gridDim.x * MT) {
    if (i + 1 < n) edge_pair_join(p.ekeyS, p.evalS, p.nbr, i, n);
    const unsigned long long k = p.ukeyS[i];
    p.uHead[i] = k != NONE && (i == 0 || p.ukeyS[i - 1] != k);
  }
}

// every corner's unknown (-1 for an unseen face); the seam edges at the first of their two sorted positions
__global__ void __launch_bounds__(MT) seams_unknown_kernel(SeamsParams p)
{
  const int n = 3 * p.T;
  for (int i = blockIdx.x * MT + threadIdx.x; i < n; i += gridDim.x * MT) {
    p.cornerUnk[p.uvalS[i]] = p.ukeyS[i] != NONE ? p.uScan[i] - 1 : -1;
    const int c = p.evalS[i], g = p.nbr[c];
    bool seam = false;
    if (g >= 0 && (i == 0 || p.ekeyS[i - 1] != p.ekeyS[i])) {
      const int a = p.view[c / 3], b = p.view[g];
      seam = a >= 0 && b >= 0 && a != b;
    }
    p.seFlag[i] = seam;
  }
}

// the smoothness key (min << 32) | max of the two unknowns of every edge of a seen face (rule 4)
__global__ void __launch_bounds__(MT) seams_smooth_keys_kernel(SeamsParams p)
{
  for (int c = blockIdx.x * MT + threadIdx.x; c < 3 * p.T; c += gridDim.x * MT) {
    const int t = c / 3, k = c - 3 * t;
    const int a = p.cornerUnk[c], b = p.cornerUnk[3 * t + (k + 1) % 3];
    p.ukey[c] = a >= 0 ? ((unsigned long long)(unsigned int)min(a, b) << 32) | (unsigned int)max(a, b) : NONE;
  }
}

__global__ void __launch_bounds__(MT) seams_smooth_heads_kernel(SeamsParams p)
{
  const int n = 3 * p.T;
  for (int i = blockIdx.x * MT + threadIdx.x; i < n; i += gridDim.x * MT) {
    const unsigned long long k = p.skeyS[i];
    p.sHead[i] = k != NONE && (i == 0 || p.skeyS[i - 1] != k);
  }
}

// Bilinear read of the atlas at (x, y), texel centres at integers, taps clamped to the chart rectangle e.
__device__ __forceinline__ double seams_bilinear(const SeamsParams &p, const int *e, double x, double y)
{
  const double x0 = floor(x), y0 = floor(y), fx = x - x0, fy = y - y0;
  const double xl = (double)e[5], xh = (double)(e[5] + e[3] - 1), yl = (double)e[6], yh = (double)(e[6] + e[4] - 1);
  const int xa = (int)fmin(fmax(x0, xl), xh), xb = (int)fmin(fmax(x0 + 1.0, xl), xh);
  const int ya = (int)fmin(fmax(y0, yl), yh), yb = (int)fmin(fmax(y0 + 1.0, yl), yh);
  const float *ra = p.atlas + (size_t)ya * p.width, *rb = p.atlas + (size_t)yb * p.width;
  const double r0 = (1.0 - fx) * (double)ra[xa] + fx * (double)ra[xb];
  const double r1 = (1.0 - fx) * (double)rb[xa] + fx * (double)rb[xb];
  return (1.0 - fy) * r0 + fy * r1;
}

// the uv of vertex w in face f (one of its corners holds it)
__device__ __forceinline__ void seams_uv_of(const SeamsParams &p, int f, int w, double &u, double &v, int &corner)
{
  int k = 0;
  while (p.tin[3 * (size_t)f + k] != w) k++;
  corner = 3 * f + k;
  u = (double)p.uv[2 * (size_t)corner];
  v = (double)p.uv[2 * (size_t)corner + 1];
}

// The two sides of the seam edge at sorted position i (rule 3): faces fs (side 0 the lower label), the uv of the ends
// P and Q on each side and their corners, and the sample count S.
struct SeamSides {
  int fs[2], cP[2], cQ[2], S;
  double uP[2], vP[2], uQ[2], vQ[2];
};

__device__ __forceinline__ void seams_edge_sides(const SeamsParams &p, int i, SeamSides &s)
{
  const unsigned long long key = p.ekeyS[i];
  const int P = (int)(key >> 32), Q = (int)(unsigned int)key;
  s.fs[0] = p.evalS[i] / 3;
  s.fs[1] = p.nbr[p.evalS[i]];
  if (p.view[s.fs[0]] > p.view[s.fs[1]]) { const int t = s.fs[0]; s.fs[0] = s.fs[1]; s.fs[1] = t; }
  double len[2];
  for (int k = 0; k < 2; k++) {
    seams_uv_of(p, s.fs[k], P, s.uP[k], s.vP[k], s.cP[k]);
    seams_uv_of(p, s.fs[k], Q, s.uQ[k], s.vQ[k], s.cQ[k]);
    const double du = s.uQ[k] - s.uP[k], dv = s.vQ[k] - s.vP[k];
    len[k] = sqrt(du * du + dv * dv);
  }
  s.S = (int)fmax(1.0, ceil(fmax(len[0], len[1])));
}

// One thread per seam edge (rule 3): its samples, the partial sums of its two ends and their keys.
__global__ void __launch_bounds__(MT) seams_sample_kernel(SeamsParams p)
{
  const int n = 3 * p.T;
  for (int i = blockIdx.x * MT + threadIdx.x; i < n; i += gridDim.x * MT) {
    if (!p.seFlag[i]) continue;
    const int e = p.seScan[i] - 1;
    SeamSides sd;
    seams_edge_sides(p, i, sd);
    const int *fs = sd.fs, *cP = sd.cP, *cQ = sd.cQ, S = sd.S;
    const double *uP = sd.uP, *vP = sd.vP, *uQ = sd.uQ, *vQ = sd.vQ;
    const int *ea = p.ctab + 8 * (size_t)p.faceChart[fs[0]], *eb = p.ctab + 8 * (size_t)p.faceChart[fs[1]];
    double sum[2][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
    for (int k = 0; k < S; k++) {
      const double t = ((double)k + 0.5) / (double)S;
      const double Ia = seams_bilinear(p, ea, uP[0] + t * (uQ[0] - uP[0]), vP[0] + t * (vQ[0] - vP[0]));
      const double Ib = seams_bilinear(p, eb, uP[1] + t * (uQ[1] - uP[1]), vP[1] + t * (vQ[1] - vP[1]));
      const double w[2] = {1.0 - t, t};
      for (int end = 0; end < 2; end++) {
        sum[end][0] = sum[end][0] + w[end] * Ia;
        sum[end][1] = sum[end][1] + w[end] * Ib;
        sum[end][2] = sum[end][2] + w[end];
      }
    }
    for (int end = 0; end < 2; end++) {
      const int j = 2 * e + end;
      const unsigned int ga = (unsigned int)p.cornerUnk[end ? cQ[0] : cP[0]],
                         gb = (unsigned int)p.cornerUnk[end ? cQ[1] : cP[1]];
      p.xkey[j] = ((unsigned long long)ga << 32) | gb;
      p.xval[j] = j;
      for (int m = 0; m < 3; m++) p.xsum[3 * (size_t)j + m] = sum[end][m];
    }
  }
}

__global__ void __launch_bounds__(MT) seams_row_heads_kernel(SeamsParams p)
{
  const int n = 2 * p.E;
  for (int j = blockIdx.x * MT + threadIdx.x; j < n; j += gridDim.x * MT)
    p.xHead[j] = j == 0 || p.xkeyS[j - 1] != p.xkeyS[j];
}

// The rows (rule 5): seam rows at [0, Rs) in (g_a, g_b) order, each the sum of its ends' partials in sorted edge order;
// smoothness rows at [Rs, Rs + Rm) in key order.  Every row's two incidences.
__global__ void __launch_bounds__(MT) seams_rows_kernel(SeamsParams p)
{
  const int n2 = 2 * p.E, n3 = 3 * p.T;
  for (int j = blockIdx.x * MT + threadIdx.x; j < n2 + n3; j += gridDim.x * MT) {
    int r, gi, gj;
    double w, d;
    if (j < n2) {
      if (!p.xHead[j]) continue;
      r = p.xScan[j] - 1;
      const unsigned long long key = p.xkeyS[j];
      double s[3] = {0.0, 0.0, 0.0};
      for (int m = j; m < n2 && p.xkeyS[m] == key; m++)
        for (int c = 0; c < 3; c++) s[c] = s[c] + p.xsum[3 * (size_t)p.xvalS[m] + c];
      const double Fa = s[0] / s[2], Fb = s[1] / s[2];
      gi = (int)(key >> 32);
      gj = (int)(unsigned int)key;
      w = 1.0;
      d = Fb - Fa;
      p.rfa[r] = Fa;
      p.rfb[r] = Fb;
    } else {
      const int i = j - n2;
      if (!p.sHead[i]) continue;
      r = p.Rs + p.sScan[i] - 1;
      const unsigned long long key = p.skeyS[i];
      gi = (int)(key >> 32);
      gj = (int)(unsigned int)key;
      w = p.smooth;
      d = 0.0;
    }
    p.ri[r] = gi;
    p.rj[r] = gj;
    p.rw[r] = w;
    p.rd[r] = d;
    p.ikey[2 * r] = gi;
    p.ival[2 * r] = 2 * r;
    p.ikey[2 * r + 1] = gj;
    p.ival[2 * r + 1] = 2 * r + 1;
  }
}

// ---- the solve (rule 6) -------------------------------------------------------------------------------------------
// The seam energy term of seam row r at offsets g (0 when g is null).
__device__ __forceinline__ double seams_energy(const SeamsParams &p, int r, const double *g)
{
  const double e = (p.rfa[r] + (g ? g[p.ri[r]] : 0.0)) - (p.rfb[r] + (g ? g[p.rj[r]] : 0.0));
  return e * e;
}

// Jacobi-PCG over N unknowns and P's x, r, z, q, diag, maxIt and totals (partA, groupA for r.r and r.z; partB, groupB
// for p.q), from rr = r.r and rz = r.z totalled to the stop: r.r <= thr, maxIt iterations, or p.q not positive.
// Returns the iteration count.  product(it, beta) writes p = z + beta p_old, q = A p and the tile partials of p.q into
// partB, and returns the p it wrote.  N, t2 and t1 come from the caller: with the loop's own copies, the solve kernels
// compile to other instructions.
template <class P, class Product>
__device__ __forceinline__ int seams_pcg(cg::grid_group &grid, const P &p, int N, double thr, double &rr, double rz,
                                         double (&t2)[2], double (&t1)[1], Product product)
{
  double beta = 0.0;
  int it = 0;
  while (it < p.maxIt && !(rr <= thr)) {
    const double *pv = product(it, beta);
    grid.sync();
    co_tree_groups<1, MT>(N, p.partB, p.groupB);
    grid.sync();
    co_tree_total<1, MT>(N, p.groupB, t1);
    if (!(t1[0] > 0.0)) break;
    const double alpha = rz / t1[0];
    // x += alpha p, r -= alpha q, z = r / diag; the totals of r.r and r.z
    co_tree_tiles<2, MT>(N, p.partA, [&](int i, double *v) {
      p.x[i] = p.x[i] + alpha * pv[i];
      const double rv = p.r[i] - alpha * p.q[i], zv = rv / p.diag[i];
      p.r[i] = rv;
      p.z[i] = zv;
      v[0] += rv * rv;
      v[1] += rv * zv;
    });
    it++;
    grid.sync();
    co_tree_groups<2, MT>(N, p.partA, p.groupA);
    grid.sync();
    co_tree_total<2, MT>(N, p.groupA, t2);
    rr = t2[0];
    beta = t2[1] / rz;
    rz = t2[1];
  }
  return it;
}

__global__ void __launch_bounds__(MT) seams_solve_kernel(SeamsParams p)
{
  cg::grid_group grid = cg::this_grid();
  const int tid = (int)(blockIdx.x * MT + threadIdx.x), nthreads = (int)gridDim.x * MT;
  const int N = p.N, R = p.Rs + p.Rm, n = 2 * R;

  // 0. every unknown's sorted incidences; its pieces of the diagonal and of b
  co_ranges(p.ikeyS, n, p.unk, tid, nthreads);
  grid.sync();
  co_pieces<2, 0, SL_PV, MT>(p.ikeyS, p.ivalS, p.pieces, n, p.unk, [&](int code, int, double *v) {
    const int r = code >> 1;
    const double wd = p.rw[r] * p.rd[r];
    v[0] = p.rw[r];
    v[1] = (code & 1) ? -wd : wd;
  });
  grid.sync();
  // 1. per unknown: diag = sum w + reg, b, x = 0, r = b, z = r / diag, p = 0; the totals of b.b and r.z; the seam
  // energy before
  co_tree_tiles<2, MT>(N, p.partA, [&](int i, double *v) {
    double G[2];
    co_gather<2, 0, SL_PV>(p.pieces, i, p.unk[i], G);
    const double dg = G[0] + p.reg, rv = G[1], zv = rv / dg;
    p.diag[i] = dg;
    p.b[i] = rv;
    p.x[i] = 0.0;
    p.r[i] = rv;
    p.z[i] = zv;
    p.p[i] = 0.0;
    v[0] += rv * rv;
    v[1] += rv * zv;
  });
  co_tree_tiles<1, MT>(p.Rs, p.partE, [&](int r, double *v) { v[0] += seams_energy(p, r, nullptr); });
  grid.sync();
  co_tree_groups<2, MT>(N, p.partA, p.groupA);
  co_tree_groups<1, MT>(p.Rs, p.partE, p.groupE);
  grid.sync();
  double t2[2], t1[1], e0[1];
  co_tree_total<2, MT>(N, p.groupA, t2);
  co_tree_total<1, MT>(p.Rs, p.groupE, e0);
  const double bb = t2[0], thr = p.tol2 * bb;
  double rr = t2[0];
  const int it = seams_pcg(grid, p, N, thr, rr, t2[1], t2, t1, [&](int, double beta) {
    // 2. the pieces of sum w p_other, p = z + beta p_old of the other unknown
    co_pieces<1, 1, SL_PV, MT>(p.ikeyS, p.ivalS, p.pieces, n, p.unk, [&](int code, int, double *v) {
      const int r = code >> 1, o = (code & 1) ? p.ri[r] : p.rj[r];
      v[0] = p.rw[r] * (p.z[o] + beta * p.p[o]);
    });
    grid.sync();
    // 3. p = z + beta p_old, q = A p = diag p - sum w p_other; the partials of p.q
    co_tree_tiles<1, MT>(N, p.partB, [&](int i, double *v) {
      double Wp[1];
      co_gather<1, 1, SL_PV>(p.pieces, i, p.unk[i], Wp);
      const double pn = p.z[i] + beta * p.p[i], qv = p.diag[i] * pn - Wp[0];
      p.p[i] = pn;
      p.q[i] = qv;
      v[0] += pn * qv;
    });
    return (const double *)p.p;
  });
  // 5. the true residual b - A x and the seam energy after; the corner offsets
  co_pieces<1, 1, SL_PV, MT>(p.ikeyS, p.ivalS, p.pieces, n, p.unk, [&](int code, int, double *v) {
    const int r = code >> 1, o = (code & 1) ? p.ri[r] : p.rj[r];
    v[0] = p.rw[r] * p.x[o];
  });
  for (int c = tid; c < 3 * p.T; c += nthreads) {
    const int g = p.cornerUnk[c];
    p.corner[c] = g >= 0 ? __double2float_rn(p.x[g]) : __int_as_float(0x7fc00000);
  }
  grid.sync();
  co_tree_tiles<1, MT>(N, p.partB, [&](int i, double *v) {
    double Wx[1];
    co_gather<1, 1, SL_PV>(p.pieces, i, p.unk[i], Wx);
    const double res = p.b[i] - (p.diag[i] * p.x[i] - Wx[0]);
    v[0] += res * res;
  });
  co_tree_tiles<1, MT>(p.Rs, p.partE, [&](int r, double *v) { v[0] += seams_energy(p, r, p.x); });
  grid.sync();
  co_tree_groups<1, MT>(N, p.partB, p.groupB);
  co_tree_groups<1, MT>(p.Rs, p.partE, p.groupE);
  grid.sync();
  double e1[1];
  co_tree_total<1, MT>(N, p.groupB, t1);
  co_tree_total<1, MT>(p.Rs, p.groupE, e1);
  if (tid == 0) {
    p.res->iters = it;
    p.res->converged = rr <= thr;
    p.res->info[0] = e0[0];
    p.res->info[1] = e1[0];
    p.res->info[2] = bb > 0.0 ? sqrt(t1[0] / bb) : 0.0;
  }
}

// ---- texels (rule 7) ----------------------------------------------------------------------------------------------
// The squared distance from (X, Y) to face f's uv triangle and the barycentric weights of the closest point: inside by
// the lower-vertex edge rule (distance 0), else the nearest of the three segments (ties to the lower edge).
__device__ __forceinline__ double seams_closest(const SeamsParams &p, int f, double X, double Y, double (&bw)[3])
{
  int id[3];
  double u[3], v[3];
  for (int k = 0; k < 3; k++) {
    id[k] = p.tin[3 * (size_t)f + k];
    u[k] = (double)p.uv[6 * (size_t)f + 2 * k];
    v[k] = (double)p.uv[6 * (size_t)f + 2 * k + 1];
  }
  const double A = (u[1] - u[0]) * (v[2] - v[0]) - (v[1] - v[0]) * (u[2] - u[0]);
  if (A != 0.0) {
    EdgeFns ef;
    edge_fns_of(id, u, v, A > 0.0 ? 1.0 : -1.0, ef);
    double w[3];
    bool in = true;
    for (int k = 0; k < 3 && in; k++) {
      w[k] = edge_fn(ef, u, v, k, X, Y);
      in = w[k] >= 0.0;
    }
    if (in) {
      const double S = (w[0] + w[1]) + w[2];
      if (S > 0.0) {
        bw[0] = w[1] / S;
        bw[1] = w[2] / S;
        bw[2] = w[0] / S;
        return 0.0;
      }
    }
  }
  double best = INFINITY;
  for (int k = 0; k < 3; k++) {
    const int k1 = (k + 1) % 3;
    const double dx = u[k1] - u[k], dy = v[k1] - v[k], l2 = dx * dx + dy * dy;
    const double t = l2 > 0.0 ? fmin(fmax(((X - u[k]) * dx + (Y - v[k]) * dy) / l2, 0.0), 1.0) : 0.0;
    const double ex = X - (u[k] + t * dx), ey = Y - (v[k] + t * dy), d2 = ex * ex + ey * ey;
    if (d2 < best) {
      best = d2;
      bw[k] = 1.0 - t;
      bw[k1] = t;
      bw[(k + 2) % 3] = 0.0;
    }
  }
  return best;
}

// One thread per seen face: every texel of its chart rectangle inside its uv box grown by padding + 1 gets atomicMin
// of (float(distance) bits << 32) | face.
__global__ void __launch_bounds__(MT) seams_raster_kernel(SeamsParams p)
{
  for (int f = blockIdx.x * MT + threadIdx.x; f < p.T; f += gridDim.x * MT) {
    if (p.view[f] < 0) continue;
    const int *e = p.ctab + 8 * (size_t)p.faceChart[f];
    const float *u = p.uv + 6 * (size_t)f;
    const double g = (double)(p.padding + 1);
    const double xlo = fmax((double)e[5], floor(fmin(fmin((double)u[0], (double)u[2]), (double)u[4])) - g);
    const double xhi = fmin((double)(e[5] + e[3] - 1), ceil(fmax(fmax((double)u[0], (double)u[2]), (double)u[4])) + g);
    const double ylo = fmax((double)e[6], floor(fmin(fmin((double)u[1], (double)u[3]), (double)u[5])) - g);
    const double yhi = fmin((double)(e[6] + e[4] - 1), ceil(fmax(fmax((double)u[1], (double)u[3]), (double)u[5])) + g);
    for (int y = (int)ylo; y <= (int)yhi; y++)
      for (int x = (int)xlo; x <= (int)xhi; x++) {
        double bw[3];
        const float d = __double2float_rn(sqrt(seams_closest(p, f, (double)x, (double)y, bw)));
        atomicMin(p.tkey + (size_t)y * p.width + x, ((unsigned long long)__float_as_uint(d) << 32) | (unsigned int)f);
      }
  }
}

// One thread per atlas texel: atlas + the winning face's interpolated corner offset (rounded to float), or a copy.
__global__ void __launch_bounds__(MT) seams_texel_kernel(SeamsParams p)
{
  const long long n = (long long)p.rows * p.width;
  unsigned long long visited = 0;
  for (long long i = blockIdx.x * (long long)MT + threadIdx.x; i < n; i += (long long)gridDim.x * MT) {
    const unsigned long long key = p.tkey[i];
    const float a = p.atlas[i];
    if (key == NONE) { p.out[i] = a; continue; }
    visited++;
    if (p.copyAll) { p.out[i] = a; continue; }
    const int f = (int)(unsigned int)key, y = (int)(i / p.width), x = (int)(i - (long long)y * p.width);
    double bw[3];
    seams_closest(p, f, (double)x, (double)y, bw);
    const float *o = p.corner + 3 * (size_t)f;
    const double off = (bw[0] * (double)o[0] + bw[1] * (double)o[1]) + bw[2] * (double)o[2];
    p.out[i] = __fadd_rn(a, __double2float_rn(off));
  }
  if (visited) atomicAdd(&p.res->texels, visited);
}

}  // namespace

// The row index of the chart table (rule 1): per atlas row y, rowList[rowStart[y], rowStart[y + 1]) the charts that
// cover it by (ox, index); rowList holds at least one entry.
static void seams_row_index(const int *charts, int numCharts, int atlasRows, std::vector<int> &rowStart,
                            std::vector<int> &rowList)
{
  rowStart.assign((size_t)atlasRows + 1, 0);
  for (int c = 0; c < numCharts; c++)
    for (int y = charts[8 * (size_t)c + 6]; y < charts[8 * (size_t)c + 6] + charts[8 * (size_t)c + 4]; y++)
      rowStart[y + 1]++;
  for (int y = 0; y < atlasRows; y++) rowStart[y + 1] += rowStart[y];
  rowList.assign(std::max(1, rowStart[atlasRows]), 0);
  std::vector<int> order(numCharts), fill(rowStart.begin(), rowStart.end() - 1);
  for (int c = 0; c < numCharts; c++) order[c] = c;
  std::stable_sort(order.begin(), order.end(),
                   [&](int a, int b) { return charts[8 * (size_t)a + 5] < charts[8 * (size_t)b + 5]; });
  for (int c : order)
    for (int y = charts[8 * (size_t)c + 6]; y < charts[8 * (size_t)c + 6] + charts[8 * (size_t)c + 4]; y++)
      rowList[fill[y]++] = c;
}

// info_out and stats_out (either may be NULL) from the call's seven counts and three info words; status 2 writes 0
// but for the status.
static void seams_report(int status, const long long (&words)[7], const double (&inf)[3], double *info,
                         long long *stats)
{
  if (info)
    for (int k = 0; k < 3; k++) info[k] = status == 2 ? 0.0 : inf[k];
  if (stats) {
    for (int k = 0; k < 7; k++) stats[k] = status == 2 ? 0 : words[k];
    stats[7] = status;
  }
}

// No face: the atlas copied, status 1.
static int seams_no_faces(const float *atlas, float *outAtlas, size_t atlasBytes, cudaStream_t st, double *info,
                          long long *stats)
{
  if (atlasBytes) CS_CUDA(cudaMemcpyAsync(outAtlas, atlas, atlasBytes, cudaMemcpyDeviceToDevice, st));
  CS_CUDA(cudaStreamSynchronize(st));
  const long long words[7] = {};
  const double inf[3] = {};
  seams_report(1, words, inf, info, stats);
  return 0;
}

// The host side of both calls up to their own stages: the row index, the scratch of the input check and the edge stage
// (and SeamsParams's pointers into it), the result words, the input check and the edge stage.  A call takes its own
// buffers from L between the constructor and alloc(); the scratch is freed on the stream when the object goes.
struct SeamsHost {
  SeamsParams &p;
  const int *charts;
  int numCharts;
  size_t resBytes;                            // the caller's result words, SeamsResult first
  void *h_res;
  cudaStream_t st;
  cudaEvent_t *tev = match_timing_events();
  std::vector<int> rowStart, rowList;
  Layout L{256};
  size_t resAt, ctabAt, rsAt, rlAt, fcAt, ekAt, ekSAt, ukAt, ukSAt, evAt, evSAt, uvAt, uvSAt, nbrAt, uhAt, usAt, sfAt,
      ssAt, cuAt;
  char *base = nullptr;
  void *temp = nullptr;
  size_t tempB = 0;

  SeamsHost(SeamsParams &p_, const float *vin, int V, const int *tin, int T, const int *faceView, const float *uv,
            const int *charts_, int numCharts_, const float *atlas, int atlasRows, int atlasWidth, int padding,
            float *outAtlas, size_t resBytes_, void *h_res_, cudaStream_t st_)
      : p(p_), charts(charts_), numCharts(numCharts_), resBytes(resBytes_), h_res(h_res_), st(st_)
  {
    p.V = V;
    p.T = T;
    p.vin = vin;
    p.tin = tin;
    p.view = faceView;
    p.uv = uv;
    p.atlas = atlas;
    p.out = outAtlas;
    p.rows = atlasRows;
    p.width = atlasWidth;
    p.padding = padding;
    seams_row_index(charts, numCharts, atlasRows, rowStart, rowList);
    const size_t C3 = 3 * (size_t)T;
    resAt = L.take(resBytes);
    ctabAt = L.take(std::max(1, numCharts) * 32ull), rsAt = L.take(rowStart.size() * 4);
    rlAt = L.take(rowList.size() * 4);
    fcAt = L.take((size_t)T * 4);
    ekAt = L.take(C3 * 8), ekSAt = L.take(C3 * 8), ukAt = L.take(C3 * 8), ukSAt = L.take(C3 * 8);
    evAt = L.take(C3 * 4), evSAt = L.take(C3 * 4), uvAt = L.take(C3 * 4), uvSAt = L.take(C3 * 4);
    nbrAt = L.take(C3 * 4);
    uhAt = L.take(C3 * 4), usAt = L.take(C3 * 4), sfAt = L.take(C3 * 4), ssAt = L.take(C3 * 4), cuAt = L.take(C3 * 4);
  }
  ~SeamsHost()
  {
    if (base) cudaFreeAsync(base, st);
  }
  char *at(size_t off) const { return base + off; }

  // The scratch, with cub's storage for the edge stage's sorts and scans and for the caller's cubBytes.
  int alloc(size_t cubBytes)
  {
    const int n3 = 3 * p.T;
    size_t tb[2] = {};
    CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb[0], (unsigned long long *)nullptr,
                                            (unsigned long long *)nullptr, (int *)nullptr, (int *)nullptr, n3, 0, 64,
                                            st));
    CS_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tb[1], (int *)nullptr, (int *)nullptr, n3, st));
    tempB = std::max(std::max(tb[0], tb[1]), cubBytes);
    const size_t tempAt = L.take(tempB);
    CS_CUDA(cudaMallocAsync((void **)&base, L.bytes, st));
    temp = at(tempAt);
    p.res = reinterpret_cast<SeamsResult *>(at(resAt));
    p.ctab = reinterpret_cast<const int *>(at(ctabAt));
    p.rowStart = reinterpret_cast<const int *>(at(rsAt));
    p.rowList = reinterpret_cast<const int *>(at(rlAt));
    p.faceChart = reinterpret_cast<int *>(at(fcAt));
    p.ekey = reinterpret_cast<unsigned long long *>(at(ekAt));
    p.ekeyS = reinterpret_cast<unsigned long long *>(at(ekSAt));
    p.ukey = reinterpret_cast<unsigned long long *>(at(ukAt));
    p.ukeyS = reinterpret_cast<unsigned long long *>(at(ukSAt));
    p.eval = reinterpret_cast<int *>(at(evAt));
    p.evalS = reinterpret_cast<int *>(at(evSAt));
    p.uval = reinterpret_cast<int *>(at(uvAt));
    p.uvalS = reinterpret_cast<int *>(at(uvSAt));
    p.nbr = reinterpret_cast<int *>(at(nbrAt));
    p.uHead = reinterpret_cast<int *>(at(uhAt));
    p.uScan = reinterpret_cast<int *>(at(usAt));
    p.seFlag = reinterpret_cast<int *>(at(sfAt));
    p.seScan = reinterpret_cast<int *>(at(ssAt));
    p.cornerUnk = reinterpret_cast<int *>(at(cuAt));
    return 0;
  }

  // the result words to the host (one synchronise)
  int readback()
  {
    CS_CUDA(cudaMemcpyAsync(h_res, p.res, resBytes, cudaMemcpyDeviceToHost, st));
    CS_CUDA(cudaStreamSynchronize(st));
    return 0;
  }

  // the count of a flag list: the last entry of its inclusive scan, into a result word
  int last(int *word, const int *scan, int n)
  {
    if (n > 0) CS_CUDA(cudaMemcpyAsync(word, scan + n - 1, 4, cudaMemcpyDeviceToDevice, st));
    return 0;
  }

  // Rule 1: the result words cleared, the chart table and its row index uploaded, the mesh and every seen face's chart
  // checked, and the words read back; bad when the input is invalid (status 2).
  int check(bool &bad)
  {
    int r;
    if (tev) CS_CUDA(cudaEventRecord(tev[0], st));
    CS_CUDA(cudaMemsetAsync(p.res, 0, resBytes, st));
    if (numCharts) CS_CUDA(cudaMemcpyAsync(at(ctabAt), charts, (size_t)numCharts * 32, cudaMemcpyHostToDevice, st));
    CS_CUDA(cudaMemcpyAsync(at(rsAt), rowStart.data(), rowStart.size() * 4, cudaMemcpyHostToDevice, st));
    CS_CUDA(cudaMemcpyAsync(at(rlAt), rowList.data(), rowList.size() * 4, cudaMemcpyHostToDevice, st));
    mesh_validate_kernel<<<grid_of(p.T), MT, 0, st>>>(p.vin, p.V, p.tin, p.T, &p.res->bad);
    seams_check_kernel<<<grid_of(p.T), MT, 0, st>>>(p);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    if ((r = readback()) < 0) return r;
    bad = static_cast<SeamsResult *>(h_res)->bad;
    return 0;
  }

  // The edges (rules 2 and 3): the adjacency, every corner's unknown and the seam edge flags and their scans.
  int edges()
  {
    const int n3 = 3 * p.T;
    if (tev) CS_CUDA(cudaEventRecord(tev[1], st));
    seams_keys_kernel<<<grid_of(3ll * p.T), MT, 0, st>>>(p);
    CS_CUDA(cub::DeviceRadixSort::SortPairs(temp, tempB, p.ekey, p.ekeyS, p.eval, p.evalS, n3, 0, 64, st));
    CS_CUDA(cub::DeviceRadixSort::SortPairs(temp, tempB, p.ukey, p.ukeyS, p.uval, p.uvalS, n3, 0, 64, st));
    seams_adjacency_kernel<<<grid_of(3ll * p.T), MT, 0, st>>>(p);
    CS_CUDA(cub::DeviceScan::InclusiveSum(temp, tempB, p.uHead, p.uScan, n3, st));
    seams_unknown_kernel<<<grid_of(3ll * p.T), MT, 0, st>>>(p);
    CS_CUDA(cub::DeviceScan::InclusiveSum(temp, tempB, p.seFlag, p.seScan, n3, st));
    count_launch(3);
    CS_CUDA(cudaGetLastError());
    return 0;
  }
};

int seams_run(const float *vin, int V, const int *tin, int T, const int *faceView, const float *uv, const int *charts,
              int numCharts, const float *atlas, int atlasRows, int atlasWidth, int padding, double smoothness,
              double regularization, int maxIterations, double tol, float *outAtlas, float *cornerOffset,
              cudaStream_t st, void *h_res, double *info, long long *stats)
{
  const size_t atlasBytes = (size_t)atlasRows * atlasWidth * 4;
  if (T == 0) return seams_no_faces(atlas, outAtlas, atlasBytes, st, info, stats);   // no seam row

  SeamsParams p{};
  SeamsHost H(p, vin, V, tin, T, faceView, uv, charts, numCharts, atlas, atlasRows, atlasWidth, padding, outAtlas,
              sizeof(SeamsResult), h_res, st);
  const size_t C3 = 3 * (size_t)T, E2 = C3, R2 = 2 * (2 * C3);   // seam ends <= 3T, rows <= 2 (3T)
  size_t tb[2] = {};
  CS_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb[0], (unsigned long long *)nullptr,
                                         (unsigned long long *)nullptr, (int)C3, 0, 64, st));
  CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb[1], (int *)nullptr, (int *)nullptr, (int *)nullptr,
                                          (int *)nullptr, (int)R2, 0, 32, st));
  const int tiles3 = (int)((C3 + CO_TREE_TILE - 1) / CO_TREE_TILE), groups3 = (tiles3 + MT - 1) / MT;

  Layout &L = H.L;
  const size_t skSAt = L.take(C3 * 8), shAt = L.take(C3 * 4), shsAt = L.take(C3 * 4);
  const size_t xkAt = L.take(E2 * 8), xkSAt = L.take(E2 * 8), xvAt = L.take(E2 * 4), xvSAt = L.take(E2 * 4),
               xhAt = L.take(E2 * 4), xsAt = L.take(E2 * 4), xsumAt = L.take(E2 * 24);
  const size_t Rmax = 2 * C3;                 // seam rows <= seam ends, smoothness rows <= corners
  const size_t riAt = L.take(Rmax * 4), rjAt = L.take(Rmax * 4), rwAt = L.take(Rmax * 8), rdAt = L.take(Rmax * 8),
               rfaAt = L.take(C3 * 8), rfbAt = L.take(C3 * 8);
  const size_t ikAt = L.take(R2 * 4), ikSAt = L.take(R2 * 4), ivAt = L.take(R2 * 4), ivSAt = L.take(R2 * 4);
  const size_t unkAt = L.take(C3 * sizeof(SeamUnk));
  const size_t vecAt = L.take(7 * C3 * 8);
  const size_t piecesAt = L.take(((R2 + CO_TILE - 1) / CO_TILE + C3) * SL_PV * 8);
  const size_t partAAt = L.take((size_t)tiles3 * 16), groupAAt = L.take((size_t)groups3 * 16),
               partBAt = L.take((size_t)tiles3 * 8), groupBAt = L.take((size_t)groups3 * 8),
               partEAt = L.take((size_t)tiles3 * 8), groupEAt = L.take((size_t)groups3 * 8);
  const size_t tkeyAt = L.take(atlasBytes * 2);
  if (const int e = H.alloc(std::max(tb[0], tb[1])); e < 0) return e;
  auto at = [&](size_t off) { return H.at(off); };

  p.corner = cornerOffset;
  p.skeyS = reinterpret_cast<unsigned long long *>(at(skSAt));
  p.sHead = reinterpret_cast<int *>(at(shAt));
  p.sScan = reinterpret_cast<int *>(at(shsAt));
  p.xkey = reinterpret_cast<unsigned long long *>(at(xkAt));
  p.xkeyS = reinterpret_cast<unsigned long long *>(at(xkSAt));
  p.xval = reinterpret_cast<int *>(at(xvAt));
  p.xvalS = reinterpret_cast<int *>(at(xvSAt));
  p.xHead = reinterpret_cast<int *>(at(xhAt));
  p.xScan = reinterpret_cast<int *>(at(xsAt));
  p.xsum = reinterpret_cast<double *>(at(xsumAt));
  p.ri = reinterpret_cast<int *>(at(riAt));
  p.rj = reinterpret_cast<int *>(at(rjAt));
  p.rw = reinterpret_cast<double *>(at(rwAt));
  p.rd = reinterpret_cast<double *>(at(rdAt));
  p.rfa = reinterpret_cast<double *>(at(rfaAt));
  p.rfb = reinterpret_cast<double *>(at(rfbAt));
  p.ikey = reinterpret_cast<int *>(at(ikAt));
  p.ikeyS = reinterpret_cast<int *>(at(ikSAt));
  p.ival = reinterpret_cast<int *>(at(ivAt));
  p.ivalS = reinterpret_cast<int *>(at(ivSAt));
  p.unk = reinterpret_cast<SeamUnk *>(at(unkAt));
  double *vec = reinterpret_cast<double *>(at(vecAt));
  p.x = vec;
  p.r = vec + C3;
  p.z = vec + 2 * C3;
  p.p = vec + 3 * C3;
  p.q = vec + 4 * C3;
  p.diag = vec + 5 * C3;
  p.b = vec + 6 * C3;
  p.pieces = reinterpret_cast<double *>(at(piecesAt));
  p.partA = reinterpret_cast<double *>(at(partAAt));
  p.groupA = reinterpret_cast<double *>(at(groupAAt));
  p.partB = reinterpret_cast<double *>(at(partBAt));
  p.groupB = reinterpret_cast<double *>(at(groupBAt));
  p.partE = reinterpret_cast<double *>(at(partEAt));
  p.groupE = reinterpret_cast<double *>(at(groupEAt));
  p.tkey = reinterpret_cast<unsigned long long *>(at(tkeyAt));
  p.smooth = smoothness;
  p.reg = regularization;
  p.tol2 = tol * tol;
  p.maxIt = maxIterations;
  void *temp = H.temp;
  size_t tempB = H.tempB;
  SeamsResult &R = *static_cast<SeamsResult *>(h_res);
  cudaEvent_t *tev = H.tev;
  const int n3 = (int)C3;

  int status = 0;
  auto run = [&]() -> int {
    int r;
    bool bad;
    if ((r = H.check(bad)) < 0) return r;
    if (bad) {
      status = 2;
      return 0;
    }
    // unknowns, adjacency, smoothness rows, seam edges
    if ((r = H.edges()) < 0) return r;
    seams_smooth_keys_kernel<<<grid_of(3ll * T), MT, 0, st>>>(p);
    CS_CUDA(cub::DeviceRadixSort::SortKeys(temp, tempB, p.ukey, p.skeyS, n3, 0, 64, st));
    seams_smooth_heads_kernel<<<grid_of(3ll * T), MT, 0, st>>>(p);
    CS_CUDA(cub::DeviceScan::InclusiveSum(temp, tempB, p.sHead, p.sScan, n3, st));
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    if ((r = H.last(&p.res->unknowns, p.uScan, n3)) < 0) return r;
    if ((r = H.last(&p.res->seamEdges, p.seScan, n3)) < 0) return r;
    if ((r = H.last(&p.res->smoothRows, p.sScan, n3)) < 0) return r;
    if ((r = H.readback()) < 0) return r;
    p.N = R.unknowns;
    p.E = R.seamEdges;
    p.Rm = R.smoothRows;
    // the seam rows
    if (tev) CS_CUDA(cudaEventRecord(tev[2], st));
    seams_sample_kernel<<<grid_of(3ll * T), MT, 0, st>>>(p);
    CS_CUDA(cub::DeviceRadixSort::SortPairs(temp, tempB, p.xkey, p.xkeyS, p.xval, p.xvalS, 2 * p.E, 0, 64, st));
    seams_row_heads_kernel<<<grid_of(2ll * p.E), MT, 0, st>>>(p);
    CS_CUDA(cub::DeviceScan::InclusiveSum(temp, tempB, p.xHead, p.xScan, 2 * p.E, st));
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    if ((r = H.last(&p.res->seamRows, p.xScan, 2 * p.E)) < 0) return r;
    if ((r = H.readback()) < 0) return r;
    p.Rs = R.seamRows;
    p.copyAll = p.Rs == 0;
    const int nInc = 2 * (p.Rs + p.Rm);
    seams_rows_kernel<<<grid_of(2ll * p.E + 3ll * T), MT, 0, st>>>(p);
    CS_CUDA(cub::DeviceRadixSort::SortPairs(temp, tempB, p.ikey, p.ikeyS, p.ival, p.ivalS, nInc, 0,
                                            radix_bits(std::max(0, p.N - 1)), st));
    CS_CUDA(cudaMemsetAsync(p.unk, 0, (size_t)p.N * sizeof(SeamUnk), st));
    count_launch();
    CS_CUDA(cudaGetLastError());
    // the solve
    if (tev) CS_CUDA(cudaEventRecord(tev[3], st));
    const int wave = coop_grid<seams_solve_kernel, MT>("cs_level_texture_seams");
    if (wave < 0) return wave;
    void *args[] = {&p};
    CS_CUDA(cudaLaunchCooperativeKernel((const void *)seams_solve_kernel, dim3(wave), dim3(MT), args, 0, st));
    count_launch();
    // the texels
    if (tev) CS_CUDA(cudaEventRecord(tev[4], st));
    CS_CUDA(cudaMemsetAsync(p.tkey, 0xff, atlasBytes * 2, st));
    seams_raster_kernel<<<grid_of(T), MT, 0, st>>>(p);
    seams_texel_kernel<<<grid_of((long long)atlasRows * atlasWidth), MT, 0, st>>>(p);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    if (tev) CS_CUDA(cudaEventRecord(tev[5], st));
    if ((r = H.readback()) < 0) return r;
    status = p.Rs == 0 ? 1 : R.converged ? 0 : 3;
    if (tev) {
      static const char *const names[5] = {"check", "unknowns", "seam rows", "solve", "texels"};
      report_stage_times(tev, names, 5, "seams timing faces=%d unknowns=%d rows=%d iterations=%d", T, p.N,
                         p.Rs + p.Rm, R.iters);
    }
    return 0;
  };
  const int r = run();
  if (r < 0) return r;
  const long long words[7] = {R.seen, R.unknowns, R.seamEdges, R.seamRows, R.smoothRows, R.iters, (long long)R.texels};
  seams_report(status, words, R.info, info, stats);
  return status == 2 ? 0 : R.unknowns;
}

size_t seams_result_bytes() { return sizeof(SeamsResult); }

// ---- local seam levelling (cs_level_texture_seams_local) -----------------------------------------------------------
// Poisson editing of the texel strips along the seams (Waechter, Moehrle & Goesele 2014, section 4.2): rule 1's check,
// the adjacency and the seam edges, rule 3's sample positions and bilinear reads and rule 7's texel keys are the
// global call's kernels and helpers above; the kernels below add the seam texels, the strip, the 5-point system, its
// solve and the output.  Every rule is stated in cudasift_b200.h at cs_level_texture_seams_local;
// tests/seam_local_oracle.py restates them in float64.
//
// Determinism: integer atomics only for counts and for the bits of max |delta| (a max of non-negative doubles is exact
// in any order).  A seam texel's targets are added in slot order (seam edge, side, k) after a stable radix sort by
// texel; a free texel's stencil in neighbour order; the totals in coop.cuh's three-level order.
namespace {

constexpr int LOC_NONE = -1;                   // a neighbour code: no neighbour (a Neumann edge)
constexpr int LOC_FIXED = -2;                  // a neighbour code: a seam or fixed texel (in the diagonal only)
constexpr int LOC_FAR = INT_MAX;               // a domain texel's hop distance before it is reached

struct LocalResult {
  SeamsResult g;                               // the words of the reused kernels (bad, seen, seamEdges)
  int samples, seamTexels, freeTexels;         // copied from the last entries of their scans
  int iters, converged;
  unsigned long long domain, maxDelta;         // maxDelta: the bits of max |delta|
  double info[2];                              // sum (f* - g)^2, the true relative residual
};

struct LocalParams {
  SeamsParams s;
  LocalResult *res;
  int n, strip, M, Ns, N, maxIt;               // n: atlas texels; M: samples; Ns: seam texels; N: free texels
  double tol2;
  int *scnt, *sscan;                           // [E] per seam edge: S, its inclusive scan
  int *skey, *skeyS, *head, *hscan;            // [2M] sample slots: texel, sorted; run heads and their scan
  double *sval, *svalS;                        // [2M] m_k
  int *stexel;                                 // [Ns] seam texels in texel order
  double *sf;                                  // [Ns] f*
  int *chart, *dA, *dB, *sidx, *uidx;          // [n] chart (-1 outside the domain), distances, seam index, free scan
  int *dist;                                   // the final distances (dA or dB)
  int4 *nb;                                    // [N] neighbour codes
  double *x, *r, *z, *pA, *pB, *q, *diag, *b;
  double *partA, *groupA, *partB, *groupB, *partE, *groupE;
};

// One thread per seam edge (rule 3): its sample count S.
__global__ void __launch_bounds__(MT) local_count_kernel(LocalParams q)
{
  const SeamsParams &p = q.s;
  for (int i = blockIdx.x * MT + threadIdx.x; i < 3 * p.T; i += gridDim.x * MT) {
    if (!p.seFlag[i]) continue;
    SeamSides sd;
    seams_edge_sides(p, i, sd);
    q.scnt[p.seScan[i] - 1] = sd.S;
  }
}

// One thread per seam edge: target m_k = 0.5 (I_a + I_b) of every sample, landed on each side's nearest texel
// (clamped to that face's chart rectangle) at slot 2 base + side S + k.
__global__ void __launch_bounds__(MT) local_sample_kernel(LocalParams q)
{
  const SeamsParams &p = q.s;
  for (int i = blockIdx.x * MT + threadIdx.x; i < 3 * p.T; i += gridDim.x * MT) {
    if (!p.seFlag[i]) continue;
    SeamSides sd;
    seams_edge_sides(p, i, sd);
    const int S = sd.S, base = 2 * (q.sscan[p.seScan[i] - 1] - S);
    const int *e[2] = {p.ctab + 8 * (size_t)p.faceChart[sd.fs[0]], p.ctab + 8 * (size_t)p.faceChart[sd.fs[1]]};
    for (int k = 0; k < S; k++) {
      const double t = ((double)k + 0.5) / (double)S;
      double X[2], Y[2];
      for (int s = 0; s < 2; s++) {
        X[s] = sd.uP[s] + t * (sd.uQ[s] - sd.uP[s]);
        Y[s] = sd.vP[s] + t * (sd.vQ[s] - sd.vP[s]);
      }
      const double m = 0.5 * (seams_bilinear(p, e[0], X[0], Y[0]) + seams_bilinear(p, e[1], X[1], Y[1]));
      for (int s = 0; s < 2; s++) {
        const int *c = e[s];
        const int tx = (int)fmin(fmax(floor(X[s] + 0.5), (double)c[5]), (double)(c[5] + c[3] - 1));
        const int ty = (int)fmin(fmax(floor(Y[s] + 0.5), (double)c[6]), (double)(c[6] + c[4] - 1));
        const int slot = base + s * S + k;
        q.skey[slot] = ty * p.width + tx;
        q.sval[slot] = m;
      }
    }
  }
}

__global__ void __launch_bounds__(MT) local_heads_kernel(LocalParams q)
{
  for (int j = blockIdx.x * MT + threadIdx.x; j < 2 * q.M; j += gridDim.x * MT)
    q.head[j] = j == 0 || q.skeyS[j - 1] != q.skeyS[j];
}

// One thread per atlas texel (rule 2): its chart (its key face's, -1 outside the domain) and distance (LOC_FAR in the
// domain, -1 outside); the domain count.
__global__ void __launch_bounds__(MT) local_domain_kernel(LocalParams q)
{
  unsigned long long inside = 0;
  for (long long i = blockIdx.x * (long long)MT + threadIdx.x; i < q.n; i += (long long)gridDim.x * MT) {
    const unsigned long long key = q.s.tkey[i];
    const bool in = key != NONE;
    q.chart[i] = in ? q.s.faceChart[(unsigned int)key] : -1;
    q.dA[i] = in ? LOC_FAR : -1;
    inside += in;
  }
  if (inside) atomicAdd(&q.res->domain, inside);
}

// One thread per run of sorted slots (rule 3): the seam texel's f*, the mean of its targets in slot order; distance 0.
__global__ void __launch_bounds__(MT) local_seam_kernel(LocalParams q)
{
  const int n = 2 * q.M;
  for (int j = blockIdx.x * MT + threadIdx.x; j < n; j += gridDim.x * MT) {
    if (!q.head[j]) continue;
    const int texel = q.skeyS[j], s = q.hscan[j] - 1;
    double sum = 0.0;
    int cnt = 0;
    for (int m = j; m < n && q.skeyS[m] == texel; m++, cnt++) sum = sum + q.svalS[m];
    assert(q.chart[texel] >= 0);               // within sqrt(2)/2 of its face, so inside its face's key box
    q.stexel[s] = texel;
    q.sf[s] = sum / (double)cnt;
    q.dA[texel] = 0;
    q.sidx[texel] = s;
  }
}

// One synchronous relaxation round (rule 4): d = min(d, d of a neighbour + 1) over the 4-neighbours of the same chart.
__global__ void __launch_bounds__(MT) local_relax_kernel(LocalParams q, const int *din, int *dout)
{
  const int W = q.s.width, H = q.s.rows;
  for (long long i = blockIdx.x * (long long)MT + threadIdx.x; i < q.n; i += (long long)gridDim.x * MT) {
    int d = din[i];
    const int c = q.chart[i];
    if (c >= 0 && d > 0) {
      const int y = (int)(i / W), x = (int)(i - (long long)y * W);
      const long long nbr[4] = {x > 0 ? i - 1 : -1, x + 1 < W ? i + 1 : -1, y > 0 ? i - W : -1, y + 1 < H ? i + W : -1};
      for (int k = 0; k < 4; k++)
        if (nbr[k] >= 0 && q.chart[nbr[k]] == c && din[nbr[k]] != LOC_FAR) d = min(d, din[nbr[k]] + 1);
    }
    dout[i] = d;
  }
}

// Rule 4: the free-texel flags (1 <= d <= stripWidth), over the spare distance buffer.
__global__ void __launch_bounds__(MT) local_flag_kernel(LocalParams q, int *flag)
{
  for (long long i = blockIdx.x * (long long)MT + threadIdx.x; i < q.n; i += (long long)gridDim.x * MT) {
    const int d = q.dist[i];
    flag[i] = d >= 1 && d <= q.strip;
  }
}

// One thread per free texel (rule 5): its neighbour codes, diagonal and right-hand side.
__global__ void __launch_bounds__(MT) local_unknowns_kernel(LocalParams q)
{
  const int W = q.s.width, H = q.s.rows;
  for (long long i = blockIdx.x * (long long)MT + threadIdx.x; i < q.n; i += (long long)gridDim.x * MT) {
    const int d = q.dist[i];
    if (!(d >= 1 && d <= q.strip)) continue;
    const int u = q.uidx[i] - 1, c = q.chart[i];
    const int y = (int)(i / W), x = (int)(i - (long long)y * W);
    const long long nbr[4] = {x > 0 ? i - 1 : -1, x + 1 < W ? i + 1 : -1, y > 0 ? i - W : -1, y + 1 < H ? i + W : -1};
    int code[4];
    int count = 0;
    double bv = 0.0;
    for (int k = 0; k < 4; k++) {
      code[k] = LOC_NONE;
      const long long j = nbr[k];
      if (j < 0 || q.chart[j] != c) continue;
      const int dj = q.dist[j];
      count++;
      if (dj >= 1 && dj <= q.strip) {
        code[k] = q.uidx[j] - 1;
      } else {
        code[k] = LOC_FIXED;
        if (dj == 0) bv = bv + (q.sf[q.sidx[j]] - (double)q.s.atlas[j]);
      }
    }
    q.nb[u] = make_int4(code[0], code[1], code[2], code[3]);
    q.diag[u] = (double)count;
    q.b[u] = bv;
  }
}

// (A v)_i = diag_i v_i - sum over free neighbours of v_j (in neighbour order), v_j = a_j + beta c_j (c may be null).
__device__ __forceinline__ double local_stencil(const LocalParams &q, int i, double vi, const double *a, const double *c,
                                               double beta)
{
  const int4 m = q.nb[i];
  const int code[4] = {m.x, m.y, m.z, m.w};
  double s = 0.0;
  for (int k = 0; k < 4; k++)
    if (code[k] >= 0) s = s + (c ? a[code[k]] + beta * c[code[k]] : a[code[k]]);
  return q.diag[i] * vi - s;
}

// Rule 6: Jacobi-PCG from delta = 0 over the free texels; four grid barriers per iteration, p double-buffered so that
// q = A p reads the neighbours' z and old p without a barrier between the update of p and the product.
__global__ void __launch_bounds__(MT) local_solve_kernel(LocalParams q)
{
  cg::grid_group grid = cg::this_grid();
  const int N = q.N, Ns = q.Ns;
  co_tree_tiles<2, MT>(N, q.partA, [&](int i, double *v) {
    const double rv = q.b[i], zv = rv / q.diag[i];
    q.x[i] = 0.0;
    q.r[i] = rv;
    q.z[i] = zv;
    q.pA[i] = 0.0;
    v[0] += rv * rv;
    v[1] += rv * zv;
  });
  co_tree_tiles<1, MT>(Ns, q.partE, [&](int s, double *v) {
    const double e = q.sf[s] - (double)q.s.atlas[q.stexel[s]];
    v[0] += e * e;
  });
  grid.sync();
  co_tree_groups<2, MT>(N, q.partA, q.groupA);
  co_tree_groups<1, MT>(Ns, q.partE, q.groupE);
  grid.sync();
  double t2[2], t1[1], e0[1];
  co_tree_total<2, MT>(N, q.groupA, t2);
  co_tree_total<1, MT>(Ns, q.groupE, e0);
  const double bb = t2[0], thr = q.tol2 * bb;
  double rr = t2[0];
  const int it = seams_pcg(grid, q, N, thr, rr, t2[1], t2, t1, [&](int it, double beta) {
    const double *pold = (it & 1) ? q.pB : q.pA;
    double *pnew = (it & 1) ? q.pA : q.pB;
    // p = z + beta p_old, q = A p; the partials of p.q
    co_tree_tiles<1, MT>(N, q.partB, [&](int i, double *v) {
      const double pn = q.z[i] + beta * pold[i], qv = local_stencil(q, i, pn, q.z, pold, beta);
      pnew[i] = pn;
      q.q[i] = qv;
      v[0] += pn * qv;
    });
    return (const double *)pnew;
  });
  // the true residual b - A x; max |x|
  unsigned long long mx = 0;
  co_tree_tiles<1, MT>(N, q.partB, [&](int i, double *v) {
    const double res = q.b[i] - local_stencil(q, i, q.x[i], q.x, nullptr, 0.0);
    v[0] += res * res;
    mx = max(mx, (unsigned long long)__double_as_longlong(fabs(q.x[i])));
  });
  if (mx) atomicMax(&q.res->maxDelta, mx);
  grid.sync();
  co_tree_groups<1, MT>(N, q.partB, q.groupB);
  grid.sync();
  co_tree_total<1, MT>(N, q.groupB, t1);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    q.res->iters = it;
    q.res->converged = rr <= thr;
    q.res->info[0] = e0[0];
    q.res->info[1] = bb > 0.0 ? sqrt(t1[0] / bb) : 0.0;
  }
}

// One thread per atlas texel (rule 7): a seam texel becomes float(f*), a free texel float(g + delta), the rest a copy.
__global__ void __launch_bounds__(MT) local_output_kernel(LocalParams q)
{
  for (long long i = blockIdx.x * (long long)MT + threadIdx.x; i < q.n; i += (long long)gridDim.x * MT) {
    const int d = q.dist[i];
    const float a = q.s.atlas[i];
    float o = a;
    if (d == 0) o = __double2float_rn(q.sf[q.sidx[i]]);
    else if (d >= 1 && d <= q.strip) o = __double2float_rn((double)a + q.x[q.uidx[i] - 1]);
    q.s.out[i] = o;
  }
}

}  // namespace

int seams_local_run(const float *vin, int V, const int *tin, int T, const int *faceView, const float *uv,
                    const int *charts, int numCharts, const float *atlas, int atlasRows, int atlasWidth, int padding,
                    int stripWidth, int maxIterations, double tol, float *outAtlas, cudaStream_t st, void *h_res,
                    double *info, long long *stats)
{
  const size_t n = (size_t)atlasRows * atlasWidth, atlasBytes = n * 4;
  if (T == 0) return seams_no_faces(atlas, outAtlas, atlasBytes, st, info, stats);   // no seam texel

  // the first allocation: the mesh stage and the texel arrays
  LocalParams q{};
  SeamsParams &p = q.s;
  SeamsHost H(p, vin, V, tin, T, faceView, uv, charts, numCharts, atlas, atlasRows, atlasWidth, padding, outAtlas,
              sizeof(LocalResult), h_res, st);
  const size_t C3 = 3 * (size_t)T;
  size_t cubB = 0;
  CS_CUDA(cub::DeviceScan::InclusiveSum(nullptr, cubB, (int *)nullptr, (int *)nullptr, (int)std::max(C3, n), st));
  Layout &L = H.L;
  const size_t scAt = L.take(C3 * 4), scsAt = L.take(C3 * 4);
  const size_t tkeyAt = L.take(n * 8), chAt = L.take(n * 4), daAt = L.take(n * 4), dbAt = L.take(n * 4),
               siAt = L.take(n * 4), uiAt = L.take(n * 4);
  if (const int e = H.alloc(cubB); e < 0) return e;
  auto at = [&](size_t off) { return H.at(off); };
  char *base2 = nullptr, *base3 = nullptr;

  q.res = reinterpret_cast<LocalResult *>(p.res);
  p.tkey = reinterpret_cast<unsigned long long *>(at(tkeyAt));
  q.scnt = reinterpret_cast<int *>(at(scAt));
  q.sscan = reinterpret_cast<int *>(at(scsAt));
  q.chart = reinterpret_cast<int *>(at(chAt));
  q.dA = reinterpret_cast<int *>(at(daAt));
  q.dB = reinterpret_cast<int *>(at(dbAt));
  q.sidx = reinterpret_cast<int *>(at(siAt));
  q.uidx = reinterpret_cast<int *>(at(uiAt));
  q.n = (int)n;
  q.strip = stripWidth;
  q.maxIt = maxIterations;
  q.tol2 = tol * tol;
  void *temp = H.temp;
  size_t tempB = H.tempB;
  LocalResult &R = *static_cast<LocalResult *>(h_res);
  cudaEvent_t *tev = H.tev;
  const int n3 = (int)C3;

  int status = 0;
  auto run = [&]() -> int {
    int r;
    bool bad;
    if ((r = H.check(bad)) < 0) return r;
    if (bad) {
      status = 2;
      return 0;
    }
    // the seam edges and their sample counts
    if ((r = H.edges()) < 0) return r;
    local_count_kernel<<<grid_of(3ll * T), MT, 0, st>>>(q);
    count_launch();
    CS_CUDA(cudaGetLastError());
    if ((r = H.last(&p.res->seamEdges, p.seScan, n3)) < 0) return r;
    if ((r = H.readback()) < 0) return r;
    p.E = R.g.seamEdges;
    CS_CUDA(cub::DeviceScan::InclusiveSum(temp, tempB, q.scnt, q.sscan, p.E, st));
    if ((r = H.last(&q.res->samples, q.sscan, p.E)) < 0) return r;
    // the domain: texel keys, charts and distances
    if (tev) CS_CUDA(cudaEventRecord(tev[2], st));
    CS_CUDA(cudaMemsetAsync(p.tkey, 0xff, n * 8, st));
    seams_raster_kernel<<<grid_of(T), MT, 0, st>>>(p);
    local_domain_kernel<<<grid_of((long long)n), MT, 0, st>>>(q);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    if ((r = H.readback()) < 0) return r;
    // the seam texels: the samples' slots sorted by texel, one run per seam texel
    if (tev) CS_CUDA(cudaEventRecord(tev[3], st));
    q.M = R.samples;
    const size_t S2 = 2 * (size_t)q.M;
    size_t sortB = 0, scanB = 0;
    CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sortB, (int *)nullptr, (int *)nullptr, (double *)nullptr,
                                            (double *)nullptr, (int)S2, 0, 32, st));
    CS_CUDA(cub::DeviceScan::InclusiveSum(nullptr, scanB, (int *)nullptr, (int *)nullptr, (int)S2, st));
    Layout L2(256);
    const size_t skAt = L2.take(S2 * 4), skSAt = L2.take(S2 * 4), hdAt = L2.take(S2 * 4), hsAt = L2.take(S2 * 4),
                 svAt = L2.take(S2 * 8), svSAt = L2.take(S2 * 8), stAt = L2.take(S2 * 4), sfvAt = L2.take(S2 * 8),
                 t2At = L2.take(std::max(sortB, scanB));
    CS_CUDA(cudaMallocAsync((void **)&base2, std::max<size_t>(L2.bytes, 256), st));
    q.skey = reinterpret_cast<int *>(base2 + skAt);
    q.skeyS = reinterpret_cast<int *>(base2 + skSAt);
    q.head = reinterpret_cast<int *>(base2 + hdAt);
    q.hscan = reinterpret_cast<int *>(base2 + hsAt);
    q.sval = reinterpret_cast<double *>(base2 + svAt);
    q.svalS = reinterpret_cast<double *>(base2 + svSAt);
    q.stexel = reinterpret_cast<int *>(base2 + stAt);
    q.sf = reinterpret_cast<double *>(base2 + sfvAt);
    void *temp2 = base2 + t2At;
    size_t temp2B = std::max(sortB, scanB);
    local_sample_kernel<<<grid_of(3ll * T), MT, 0, st>>>(q);
    CS_CUDA(cub::DeviceRadixSort::SortPairs(temp2, temp2B, q.skey, q.skeyS, q.sval, q.svalS, (int)S2, 0,
                                            radix_bits((long long)n - 1), st));
    local_heads_kernel<<<grid_of((long long)S2), MT, 0, st>>>(q);
    CS_CUDA(cub::DeviceScan::InclusiveSum(temp2, temp2B, q.head, q.hscan, (int)S2, st));
    local_seam_kernel<<<grid_of((long long)S2), MT, 0, st>>>(q);
    count_launch(3);
    CS_CUDA(cudaGetLastError());
    if ((r = H.last(&q.res->seamTexels, q.hscan, (int)S2)) < 0) return r;
    // the strip: stripWidth relaxation rounds, the free texels numbered in atlas order
    if (tev) CS_CUDA(cudaEventRecord(tev[4], st));
    for (int k = 0; k < stripWidth; k++)
      local_relax_kernel<<<grid_of((long long)n), MT, 0, st>>>(q, (k & 1) ? q.dB : q.dA, (k & 1) ? q.dA : q.dB);
    q.dist = (stripWidth & 1) ? q.dB : q.dA;
    int *flag = (stripWidth & 1) ? q.dA : q.dB;
    local_flag_kernel<<<grid_of((long long)n), MT, 0, st>>>(q, flag);
    CS_CUDA(cub::DeviceScan::InclusiveSum(temp, tempB, flag, q.uidx, (int)n, st));
    count_launch(stripWidth + 1);
    CS_CUDA(cudaGetLastError());
    if ((r = H.last(&q.res->freeTexels, q.uidx, (int)n)) < 0) return r;
    if ((r = H.readback()) < 0) return r;
    q.Ns = R.seamTexels;
    q.N = R.freeTexels;
    // the system and its solve
    if (tev) CS_CUDA(cudaEventRecord(tev[5], st));
    const size_t N = (size_t)q.N, Ns = (size_t)q.Ns;
    const size_t tilesN = (N + CO_TREE_TILE - 1) / CO_TREE_TILE, groupsN = (tilesN + MT - 1) / MT;
    const size_t tilesS = (Ns + CO_TREE_TILE - 1) / CO_TREE_TILE, groupsS = (tilesS + MT - 1) / MT;
    Layout L3(256);
    const size_t nbAt = L3.take(N * 16), vecAt = L3.take(8 * N * 8),
                 paAt = L3.take(tilesN * 16), gaAt = L3.take(groupsN * 16), pbAt = L3.take(tilesN * 8),
                 gbAt = L3.take(groupsN * 8), peAt = L3.take(tilesS * 8), geAt = L3.take(groupsS * 8);
    CS_CUDA(cudaMallocAsync((void **)&base3, std::max<size_t>(L3.bytes, 256), st));
    q.nb = reinterpret_cast<int4 *>(base3 + nbAt);
    double *vec = reinterpret_cast<double *>(base3 + vecAt);
    q.x = vec;
    q.r = vec + N;
    q.z = vec + 2 * N;
    q.pA = vec + 3 * N;
    q.pB = vec + 4 * N;
    q.q = vec + 5 * N;
    q.diag = vec + 6 * N;
    q.b = vec + 7 * N;
    q.partA = reinterpret_cast<double *>(base3 + paAt);
    q.groupA = reinterpret_cast<double *>(base3 + gaAt);
    q.partB = reinterpret_cast<double *>(base3 + pbAt);
    q.groupB = reinterpret_cast<double *>(base3 + gbAt);
    q.partE = reinterpret_cast<double *>(base3 + peAt);
    q.groupE = reinterpret_cast<double *>(base3 + geAt);
    local_unknowns_kernel<<<grid_of((long long)n), MT, 0, st>>>(q);
    count_launch();
    CS_CUDA(cudaGetLastError());
    const int wave = coop_grid<local_solve_kernel, MT>("cs_level_texture_seams_local");
    if (wave < 0) return wave;
    void *args[] = {&q};
    CS_CUDA(cudaLaunchCooperativeKernel((const void *)local_solve_kernel, dim3(wave), dim3(MT), args, 0, st));
    count_launch();
    // the output
    if (tev) CS_CUDA(cudaEventRecord(tev[6], st));
    local_output_kernel<<<grid_of((long long)n), MT, 0, st>>>(q);
    count_launch();
    CS_CUDA(cudaGetLastError());
    if (tev) CS_CUDA(cudaEventRecord(tev[7], st));
    if ((r = H.readback()) < 0) return r;
    status = q.Ns == 0 ? 1 : R.converged ? 0 : 3;
    if (tev) {
      static const char *const names[7] = {"check", "seam edges", "domain", "seam texels", "strip", "solve",
                                           "output"};
      report_stage_times(tev, names, 7, "seams local timing faces=%d seam texels=%d free texels=%d iterations=%d", T,
                         q.Ns, q.N, R.iters);
    }
    return 0;
  };
  const int r = run();
  if (base3) cudaFreeAsync(base3, st);
  if (base2) cudaFreeAsync(base2, st);
  if (r < 0) return r;
  double inf[3] = {R.info[0], R.info[1], 0.0};
  const unsigned long long bits = R.maxDelta;
  std::memcpy(&inf[2], &bits, 8);
  const long long words[7] = {R.g.seen, R.g.seamEdges, R.samples, R.seamTexels, R.freeTexels, (long long)R.domain,
                              R.iters};
  seams_report(status, words, inf, info, stats);
  return status == 2 ? 0 : R.freeTexels;
}

size_t seams_local_result_bytes() { return sizeof(LocalResult); }

}  // namespace cs
