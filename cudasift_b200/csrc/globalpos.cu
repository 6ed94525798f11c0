// globalpos.cu -- global positioning of camera centres and track points with known rotations (cs_global_positioning,
// GLOMAP's BATA residual on points).  The rules (used observations, the residual, the per-observation scale, the loss,
// Levenberg-Marquardt, the eliminations, the gauge, the outputs and the summation orders) are stated in
// cudasift_b200.h at cs_global_positioning; tests/globalpos_oracle.py restates them in float64.
//
// Three counted launches, whatever the sizes and iteration counts, laid out as bundle.cu's:
//   1. gp_count_kernel: per track, its used observations (0 when fewer than 2) and the integer statistics
//   2. (cub scan of the counts) gp_fill_kernel: the used observations in track order, then member order, their world
//      rays and a key (image) per observation
//   3. (cub stable radix sort of (image, observation)) gp_kernel: one cooperative launch runs the whole LM loop
// The camera block is 3 wide and the per-observation scale is eliminated inside its own 7 x 7 block, so this is a
// kernel of its own rather than an instantiation of bundle_kernel.  Every floating-point sum has a fixed order that
// depends on the data only (coop.cuh): per point, a thread over its observations in order; per camera, the pieces of the
// sorted observations' tiles; totals over tiles of 256 tracks or 32 cameras.  No floating-point atomics; every branch
// around a grid barrier is taken on values every CTA computes from the same words.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <cooperative_groups.h>
#include <cub/cub.cuh>
#include <math_constants.h>

#include "common.cuh"
#include "coop.cuh"

namespace cg = cooperative_groups;

namespace cs {

namespace {

constexpr int GP_THREADS = 256;
constexpr int GP_PV = 19;            // a camera piece: sum P (6), sum w^2 s^2, sum beta (3), sum P q (3), Schur term (6)
constexpr int GP_CP = 3;             // camera tile partial slots: r.r (b~.b~), r.z, p.S p
constexpr double GP_SMIN = 1e-6;     // the lower bound of every scale s

// A used observation: its track, image, world ray; the scale (current, candidate); the linearisation (d = X - c,
// r = v - s d, w2 = rho') and, per LM iteration, the damped h, P and beta.
struct GpObs {
  int k, a;
  double v[3];
  double s, sc;
  double d[3], r[3], w2, h;
  double P[6], beta[3];
};

// A camera: its rotation and intrinsics (the rays), its record set; the centre (current, candidate), the damped U, the
// preconditioner factor, the CG vectors and its sorted observations [start, end).
struct GpCam {
  double K[6], R[9];
  const SiftPoint *pts;
  int n, hasR;
  double c[3], cc[3];
  double U[6], L[6];
  double x[3], r[3], z[3], p[3], q[3];
  int start, end, free, pad;
};

// A track's point: current, candidate; the damped V factor, b_X, V^-1 b_X and the CG scratch.
struct GpPt {
  double X[3], Xc[3];
  double L[6];
  double b[3], q[3], y[3];
};

static_assert(sizeof(GpObs) == 184 && sizeof(GpCam) == 416 && sizeof(GpPt) == 168, "the header states the scratch");

struct GpResult {
  double cost[2];
  double scale;
  unsigned long long stats[8];
  unsigned long long accepted;
};

struct GpParams {
  GpCam *cams;
  GpPt *pts;
  const int *offsets;
  const int2 *members;
  const unsigned char *use;
  double *points;
  int *cnt, *start;
  GpObs *obs;
  int *keys, *vals;
  const int *keysS, *order;
  double *pieces, *camPart, *ptPart;
  unsigned int *flags;
  double *trace;
  GpResult *res;
  double tol2, c2;
  unsigned long long seed;
  int numImages, numTracks, numMembers, maxIterations, maxLinear, loss, refImage;
};

// ---- small helpers ----------------------------------------------------------------------------------------------

// a packed symmetric 3 x 3 (upper, row by row) as a full matrix
__device__ __forceinline__ void gp_full(const double *A, double (&F)[3][3])
{
  F[0][0] = A[0]; F[0][1] = F[1][0] = A[1]; F[0][2] = F[2][0] = A[2];
  F[1][1] = A[3]; F[1][2] = F[2][1] = A[4]; F[2][2] = A[5];
}

// y = A x for a packed symmetric 3 x 3 A
__device__ __forceinline__ void gp_symv(const double *A, const double *x, double *y)
{
  y[0] = A[0] * x[0] + A[1] * x[1] + A[2] * x[2];
  y[1] = A[1] * x[0] + A[3] * x[1] + A[4] * x[2];
  y[2] = A[2] * x[0] + A[4] * x[1] + A[5] * x[2];
}

// The start draw: component j of item i of kind (0 centres, 1 points), uniform in [-1, 1).
__device__ __forceinline__ double gp_draw(unsigned long long seed, int kind, int i, int j)
{
  const unsigned long long x =
      vp_splitmix64(seed + 0x9E3779B97F4A7C15ull * ((((unsigned long long)kind << 32) | (unsigned)i) * 3 + j));
  return 2.0 * ((double)(x >> 11) * 0x1.0p-53) - 1.0;
}

// The used observations of track k (f(m, a, x, y, j)); -1 for a malformed track.
template <class F>
__device__ __forceinline__ int gp_used(const GpParams &p, int k, int &invalid, F &&f)
{
  const int lo = p.offsets[k], hi = p.offsets[k + 1];
  if (lo < 0 || hi < lo || hi > p.numMembers) return -1;
  int used = 0;
  invalid = 0;
  for (int m = lo; m < hi; m++) {
    float x, y;
    const int2 af = p.members[m];
    if (!tr_member(p.cams, p.numImages, af, x, y)) { invalid++; continue; }
    if (!p.cams[af.x].hasR || (p.use && !p.use[m])) continue;
    f(m, af.x, x, y, used);
    used++;
  }
  return used;
}

__global__ void __launch_bounds__(GP_THREADS) gp_count_kernel(GpParams p)
{
  co_count(p, blockIdx.x * GP_THREADS + threadIdx.x, [&](int k, int &invalid) {
    return gp_used(p, k, invalid, [](int, int, float, float, int) {});
  });
}

__global__ void __launch_bounds__(GP_THREADS) gp_fill_kernel(GpParams p)
{
  const int i = blockIdx.x * GP_THREADS + threadIdx.x;
  const int N = p.start[p.numTracks];
  if (i >= N && i < p.numMembers) {
    p.keys[i] = p.numImages;
    p.vals[i] = i;
  }
  if (i >= p.numTracks || p.cnt[i] == 0) return;
  const int k = i, s = p.start[k];
  int invalid = 0;
  gp_used(p, k, invalid, [&](int, int a, float x, float y, int j) {
    const GpCam &c = p.cams[a];
    double u, v;
    vp_calibrate(c.K, (double)x, (double)y, u, v);
    const double b[3] = {u, v, 1.0};
    double w[3];
#pragma unroll
    for (int q = 0; q < 3; q++) w[q] = c.R[q] * b[0] + c.R[3 + q] * b[1] + c.R[6 + q] * b[2];   // R^T b
    const double n = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    GpObs &o = p.obs[s + j];
    o.k = k;
    o.a = a;
#pragma unroll
    for (int q = 0; q < 3; q++) o.v[q] = w[q] / n;
    o.s = 1.0;
    p.keys[s + j] = a;
    p.vals[s + j] = s + j;
  });
}

// ---- the cooperative kernel ---------------------------------------------------------------------------------------

// The observations of track k at the current (or candidate) parameters: d, r and rho' stored (unless cand); the cost.
__device__ __forceinline__ double gp_relinearise(const GpParams &p, int k, int s, int e, bool cand, bool store)
{
  const GpPt &pt = p.pts[k];
  double cost = 0.0;
  for (int o = s; o < e; o++) {
    GpObs &ob = p.obs[o];
    const GpCam &c = p.cams[ob.a];
    const double sc = cand ? ob.sc : ob.s;
    double d[3], r[3];
#pragma unroll
    for (int q = 0; q < 3; q++) {
      d[q] = (cand ? pt.Xc[q] : pt.X[q]) - (cand ? c.cc[q] : c.c[q]);
      r[q] = ob.v[q] - sc * d[q];
    }
    const double s2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    double w2 = 1.0;
    cost += p.loss ? vp_loss(p.loss, p.c2, s2, &w2) : s2;
    if (store) {
#pragma unroll
      for (int q = 0; q < 3; q++) { ob.d[q] = d[q]; ob.r[q] = r[q]; }
      ob.w2 = w2;
    }
  }
  return cost;
}

__global__ void __launch_bounds__(GP_THREADS) gp_kernel(GpParams p)
{
  cg::grid_group grid = cg::this_grid();
  const int tid = (int)(blockIdx.x * GP_THREADS + threadIdx.x), nthreads = (int)gridDim.x * GP_THREADS;
  const int lane = (int)threadIdx.x & 31, warpG = tid >> 5, numWarps = nthreads >> 5;
  const int C = p.numImages, N = p.start[p.numTracks];
  const int camTiles = (C + 31) / 32, ptTiles = (p.numTracks + GP_THREADS - 1) / GP_THREADS;

  // 0. every camera's sorted range and its start centre; every point's start; the linearisation and cost at the start
  co_ranges(p.keysS, N, p.cams, tid, nthreads);
  for (int a = tid; a < C; a += nthreads) {
    GpCam &c = p.cams[a];
#pragma unroll
    for (int q = 0; q < 3; q++) c.c[q] = a == p.refImage ? 0.0 : gp_draw(p.seed, 0, a, q);
  }
  for (int k = tid; k < p.numTracks; k += nthreads)
#pragma unroll
    for (int q = 0; q < 3; q++) p.pts[k].X[q] = gp_draw(p.seed, 1, k, q);
  grid.sync();
  for (int a = tid; a < C; a += nthreads) {
    GpCam &c = p.cams[a];
    c.free = c.end > c.start && a != p.refImage;
    if (c.end > c.start) atomicAdd(&p.res->stats[5], 1ull);
  }
  co_per_track<1, GP_THREADS>(p.start, p.numTracks, p.ptPart, [&](int k, int s, int e, double *v) { v[0] = gp_relinearise(p, k, s, e, false, true); });
  grid.sync();
  double cost;
  {
    double t[1];
    co_totals<1>(p.ptPart, ptTiles, 1, t);
    cost = t[0];
  }
  const double cost0 = cost;
  double lam = 1e-3;
  unsigned long long accepted = 0, lmIters = 0, cgTotal = 0;

  for (int it = 0; it < p.maxIterations && N > 0; it++) {
    lmIters++;
    // A. per observation: s eliminated in its 7 x 7 block (h, P, beta); per point: V* by Cholesky, b_X, q = V*^-1 b_X
    co_per_track<0, GP_THREADS>(p.start, p.numTracks, nullptr, [&](int k, int s, int e, double *) {
      double V[6] = {0, 0, 0, 0, 0, 0}, b[3] = {0, 0, 0}, dg = 0.0;
      for (int o = s; o < e; o++) {
        GpObs &ob = p.obs[o];
        const double w2 = ob.w2, sv = ob.s, *d = ob.d, *r = ob.r;
        const double dd2 = w2 * (d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), h = dd2 + vp_damping(dd2, lam);
        const double a2 = w2 * sv * sv, f = w2 / h, dr = d[0] * r[0] + d[1] * r[1] + d[2] * r[2];
        int n = 0;
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
          for (int j = i; j < 3; j++) ob.P[n++] = a2 * ((i == j ? 1.0 : 0.0) - f * d[i] * d[j]);
#pragma unroll
        for (int i = 0; i < 3; i++) ob.beta[i] = w2 * sv * (r[i] - f * d[i] * dr);
        ob.h = h;
#pragma unroll
        for (int j = 0; j < 6; j++) V[j] += ob.P[j];
#pragma unroll
        for (int i = 0; i < 3; i++) b[i] += ob.beta[i];
        dg += a2;
      }
      const double dd = vp_damping(dg, lam);
      V[0] += dd; V[3] += dd; V[5] += dd;
      GpPt &pt = p.pts[k];
      double Vf[3][3];
      gp_full(V, Vf);
      if (!vp_chol<3>(Vf, pt.L)) { atomicOr(&p.flags[it], 1u); return; }
      double q[3];
      vp_chol_solve<3>(pt.L, b, q);
#pragma unroll
      for (int i = 0; i < 3; i++) { pt.b[i] = b[i]; pt.q[i] = q[i]; }
    });
    grid.sync();
    unsigned int fail = *(volatile unsigned int *)&p.flags[it];

    // B. the camera pieces: sum P, sum w^2 s^2, sum beta, sum P q and the Schur term P_o V*^-1 W_ak
    if (!fail)
      co_pieces<GP_PV, 0, GP_PV, GP_THREADS>(p.keysS, p.order, p.pieces, N, p.cams, [&](int o, int a, double *v) {
        const GpObs &ob = p.obs[o];
        const GpPt &pt = p.pts[ob.k];
#pragma unroll
        for (int j = 0; j < 6; j++) v[j] = ob.P[j];
        v[6] = ob.w2 * ob.s * ob.s;
#pragma unroll
        for (int i = 0; i < 3; i++) v[7 + i] = ob.beta[i];
        gp_symv(ob.P, pt.q, v + 10);
        double Wa[6] = {0, 0, 0, 0, 0, 0};
        for (int u = p.start[ob.k]; u < p.start[ob.k + 1]; u++)
          if (p.obs[u].a == a)
#pragma unroll
            for (int j = 0; j < 6; j++) Wa[j] += p.obs[u].P[j];
        double Y[3][3], col[3];                                // Y = V*^-1 Wa (column by column)
#pragma unroll
        for (int j = 0; j < 3; j++) {
          const double w[3] = {Wa[j == 0 ? 0 : j == 1 ? 1 : 2], Wa[j == 0 ? 1 : j == 1 ? 3 : 4],
                               Wa[j == 0 ? 2 : j == 1 ? 4 : 5]};
          vp_chol_solve<3>(pt.L, w, col);
#pragma unroll
          for (int i = 0; i < 3; i++) Y[i][j] = col[i];
        }
        double Pf[3][3];
        gp_full(ob.P, Pf);
        int n = 13;
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
          for (int j = i; j < 3; j++) v[n++] = Pf[i][0] * Y[0][j] + Pf[i][1] * Y[1][j] + Pf[i][2] * Y[2][j];
      });
    grid.sync();

    // C. per camera (a lane each): U*, b~ = -sum beta + sum P q, the preconditioner U* - T by Cholesky; CG's start
    if (!fail)
      for (int w = warpG; w < camTiles; w += numWarps) {
        const int a = w * 32 + lane;
        double d[2] = {0.0, 0.0};
        if (a < C) {
          GpCam &c = p.cams[a];
          double G[GP_PV];
          co_gather<GP_PV, 0, GP_PV>(p.pieces, a, c, G);
          const double dd = vp_damping(G[6], lam);
          double U[6], M[6];
#pragma unroll
          for (int j = 0; j < 6; j++) {
            const bool diag = j == 0 || j == 3 || j == 5;
            U[j] = c.free ? G[j] + (diag ? dd : 0.0) : (diag ? 1.0 : 0.0);
            M[j] = c.free ? U[j] - G[13 + j] : U[j];
            c.U[j] = U[j];
          }
          double Mf[3][3];
          gp_full(M, Mf);
          if (!vp_chol<3>(Mf, c.L)) {
            atomicOr(&p.flags[it], 1u);
          } else {
            double r[3], z[3];
#pragma unroll
            for (int i = 0; i < 3; i++) r[i] = c.free ? -G[7 + i] + G[10 + i] : 0.0;
            vp_chol_solve<3>(c.L, r, z);
#pragma unroll
            for (int i = 0; i < 3; i++) {
              c.x[i] = 0.0; c.r[i] = r[i]; c.z[i] = z[i]; c.p[i] = 0.0;
              d[0] += r[i] * r[i];
              d[1] += r[i] * z[i];
            }
          }
        }
        co_warp_partial<2>(d, p.camPart + GP_CP * (size_t)w);
      }
    grid.sync();
    fail = *(volatile unsigned int *)&p.flags[it];

    // D-G. block-Jacobi PCG on S dc = b~ from dc = 0 (S p = U* p - sum_o P_o y_k, y_k = V*^-1 sum_o P_o p_a)
    int cgIt = 0;
    if (!fail) {
      double t2[2];
      co_totals<2>(p.camPart, camTiles, GP_CP, t2);
      const double thr = p.tol2 * t2[0];
      double rr = t2[0], rz = t2[1], beta = 0.0;
      while (cgIt < p.maxLinear && !(rr <= thr)) {
        co_per_track<0, GP_THREADS>(p.start, p.numTracks, nullptr, [&](int k, int s, int e, double *) {
          double h[3] = {0.0, 0.0, 0.0};
          for (int o = s; o < e; o++) {
            const GpObs &ob = p.obs[o];
            const GpCam &c = p.cams[ob.a];
            const double pe[3] = {fma(beta, c.p[0], c.z[0]), fma(beta, c.p[1], c.z[1]), fma(beta, c.p[2], c.z[2])};
            double t[3];
            gp_symv(ob.P, pe, t);
#pragma unroll
            for (int i = 0; i < 3; i++) h[i] += t[i];
          }
          vp_chol_solve<3>(p.pts[k].L, h, p.pts[k].y);
        });
        grid.sync();
        co_pieces<3, 0, GP_PV, GP_THREADS>(p.keysS, p.order, p.pieces, N, p.cams, [&](int o, int, double *v) { gp_symv(p.obs[o].P, p.pts[p.obs[o].k].y, v); });
        grid.sync();
        for (int w = warpG; w < camTiles; w += numWarps) {
          const int a = w * 32 + lane;
          double d[1] = {0.0};
          if (a < C) {
            GpCam &c = p.cams[a];
            double Wy[3], pn[3], Up[3];
            co_gather<3, 0, GP_PV>(p.pieces, a, c, Wy);
#pragma unroll
            for (int i = 0; i < 3; i++) pn[i] = fma(beta, c.p[i], c.z[i]);
            gp_symv(c.U, pn, Up);
#pragma unroll
            for (int i = 0; i < 3; i++) {
              const double q = c.free ? Up[i] - Wy[i] : 0.0;
              c.p[i] = pn[i];
              c.q[i] = q;
              d[0] += pn[i] * q;
            }
          }
          co_warp_partial<1>(d, p.camPart + GP_CP * (size_t)w + 2);
        }
        grid.sync();
        double pq[1];
        co_totals<1>(p.camPart + 2, camTiles, GP_CP, pq);
        if (!(pq[0] > 0.0)) break;
        const double alpha = rz / pq[0];
        for (int w = warpG; w < camTiles; w += numWarps) {
          const int a = w * 32 + lane;
          double d[2] = {0.0, 0.0};
          if (a < C) {
            GpCam &c = p.cams[a];
            double r[3], z[3];
#pragma unroll
            for (int i = 0; i < 3; i++) {
              c.x[i] = fma(alpha, c.p[i], c.x[i]);
              r[i] = fma(-alpha, c.q[i], c.r[i]);
              c.r[i] = r[i];
            }
            vp_chol_solve<3>(c.L, r, z);
#pragma unroll
            for (int i = 0; i < 3; i++) {
              c.z[i] = z[i];
              d[0] += r[i] * r[i];
              d[1] += r[i] * z[i];
            }
          }
          co_warp_partial<2>(d, p.camPart + GP_CP * (size_t)w);
        }
        cgIt++;
        grid.sync();
        co_totals<2>(p.camPart, camTiles, GP_CP, t2);
        rr = t2[0];
        beta = t2[1] / rz;
        rz = t2[1];
      }
    }
    cgTotal += cgIt;

    // H. back-substitution: dX = V*^-1 (b_X + sum P dc), ds = w^2 (d.r - s d.(dX - dc)) / h, s >= GP_SMIN; candidates
    double cand[1] = {CUDART_NAN};
    if (!fail) {
      for (int a = tid; a < C; a += nthreads) {
        GpCam &c = p.cams[a];
#pragma unroll
        for (int i = 0; i < 3; i++) c.cc[i] = c.free ? c.c[i] + c.x[i] : c.c[i];
      }
      co_per_track<0, GP_THREADS>(p.start, p.numTracks, nullptr, [&](int k, int s, int e, double *) {
        GpPt &pt = p.pts[k];
        double h[3] = {pt.b[0], pt.b[1], pt.b[2]}, dX[3];
        for (int o = s; o < e; o++) {
          const GpCam &c = p.cams[p.obs[o].a];
          double dc[3] = {c.free ? c.x[0] : 0.0, c.free ? c.x[1] : 0.0, c.free ? c.x[2] : 0.0}, t[3];
          gp_symv(p.obs[o].P, dc, t);
#pragma unroll
          for (int i = 0; i < 3; i++) h[i] += t[i];
        }
        vp_chol_solve<3>(pt.L, h, dX);
#pragma unroll
        for (int i = 0; i < 3; i++) pt.Xc[i] = pt.X[i] + dX[i];
        for (int o = s; o < e; o++) {
          GpObs &ob = p.obs[o];
          const GpCam &c = p.cams[ob.a];
          double dd = 0.0, dr = 0.0;
#pragma unroll
          for (int i = 0; i < 3; i++) {
            dd += ob.d[i] * (dX[i] - (c.free ? c.x[i] : 0.0));
            dr += ob.d[i] * ob.r[i];
          }
          ob.sc = fmax(ob.s + ob.w2 * (dr - ob.s * dd) / ob.h, GP_SMIN);
        }
      });
      grid.sync();
      co_per_track<1, GP_THREADS>(p.start, p.numTracks, p.ptPart, [&](int k, int s, int e, double *v) { v[0] = gp_relinearise(p, k, s, e, true, false); });
      grid.sync();
      co_totals<1>(p.ptPart, ptTiles, 1, cand);
    }

    // J. accept or reject
    const bool accept = !fail && cand[0] < cost;
    if (tid == 0) {
      double *tr = p.trace + 4 * (size_t)it;
      tr[0] = fail ? CUDART_NAN : cand[0];
      tr[1] = lam;
      tr[2] = (double)cgIt;
      tr[3] = accept ? 1.0 : 0.0;
    }
    if (accept) {
      const bool stop = cost - cand[0] <= 1e-10 * cost;
      cost = cand[0];
      lam /= 10.0;
      accepted++;
      for (int a = tid; a < C; a += nthreads)
#pragma unroll
        for (int i = 0; i < 3; i++) p.cams[a].c[i] = p.cams[a].cc[i];
      co_per_track<0, GP_THREADS>(p.start, p.numTracks, nullptr, [&](int k, int s, int e, double *) {
        GpPt &pt = p.pts[k];
#pragma unroll
        for (int i = 0; i < 3; i++) pt.X[i] = pt.Xc[i];
        for (int o = s; o < e; o++) p.obs[o].s = p.obs[o].sc;
      });
      grid.sync();
      co_per_track<0, GP_THREADS>(p.start, p.numTracks, nullptr, [&](int k, int s, int e, double *) { gp_relinearise(p, k, s, e, false, true); });
      grid.sync();
      if (stop) break;
    } else {
      lam *= 10.0;
      if (lam > 1e16) break;
    }
  }

  // K. the gauge: scale = sqrt(mean |c_a|^2 over the positioned cameras) (tiles of 32 cameras); the points
  for (int w = warpG; w < camTiles; w += numWarps) {
    const int a = w * 32 + lane;
    double d[2] = {0.0, 0.0};
    if (a < C && p.cams[a].end > p.cams[a].start) {
      const double *c = p.cams[a].c;
      d[0] = c[0] * c[0] + c[1] * c[1] + c[2] * c[2];
      d[1] = 1.0;
    }
    co_warp_partial<2>(d, p.camPart + GP_CP * (size_t)w);
  }
  grid.sync();
  double t2[2];
  co_totals<2>(p.camPart, camTiles, GP_CP, t2);
  const double rms = t2[1] > 0.0 ? sqrt(t2[0] / t2[1]) : 0.0;
  const double scale = rms > 0.0 && isfinite(rms) ? rms : 1.0;
  for (int k = tid; k < p.numTracks; k += nthreads) {
    const bool has = p.start[k + 1] > p.start[k];
#pragma unroll
    for (int i = 0; i < 3; i++) p.points[3 * (size_t)k + i] = has ? p.pts[k].X[i] / scale : CUDART_NAN;
  }
  if (tid == 0) {
    p.res->cost[0] = cost0;
    p.res->cost[1] = cost;
    p.res->scale = scale;
    p.res->accepted = accepted;
    p.res->stats[6] = lmIters;
    p.res->stats[7] = cgTotal;
  }
}

size_t gp_host_layout(int numImages, int maxIterations, size_t *bytes)
{
  Layout H(256);
  H.take(sizeof(GpResult));
  H.take((size_t)maxIterations * 4 * sizeof(double));
  const size_t camAt = H.take((size_t)numImages * sizeof(GpCam));
  if (bytes) *bytes = H.bytes;
  return camAt;
}

}  // namespace

int globalpos_enqueue(DeviceCtx &c, const cs_match_set *sets, int numImages, const double *Ks, const double *Rs,
                      const int *offsets, int numTracks, const int *members, int numMembers, const unsigned char *use,
                      int refImage, unsigned long long seed, int loss, double lossScale, int maxIterations,
                      int maxLinearIterations, double linearTol, double *points)
{
  const int M = numMembers, T = numTracks, C = numImages;
  const int tiles = idivup(M, CO_TILE);
  const int bits = radix_bits(C);                                  // every key, the sentinel C included
  size_t scanBytes = 0, sortBytes = 0;
  CS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scanBytes, (int *)nullptr, (int *)nullptr, T + 1, c.stream));
  CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sortBytes, (int *)nullptr, (int *)nullptr, (int *)nullptr,
                                          (int *)nullptr, std::max(M, 1), 0, bits, c.stream));
  Layout L(256);
  const size_t resAt = L.take(sizeof(GpResult)), traceAt = L.take((size_t)maxIterations * 4 * sizeof(double));
  const size_t flagsAt = L.take((size_t)std::max(maxIterations, 1) * sizeof(unsigned int)), zeroEnd = L.bytes;
  const size_t camAt = L.take((size_t)C * sizeof(GpCam)), ptAt = L.take((size_t)T * sizeof(GpPt));
  const size_t cntAt = L.take(((size_t)T + 1) * sizeof(int)), startAt = L.take(((size_t)T + 1) * sizeof(int));
  const size_t obsAt = L.take((size_t)M * sizeof(GpObs));
  const size_t keysAt = L.take((size_t)M * sizeof(int)), valsAt = L.take((size_t)M * sizeof(int));
  const size_t keysSAt = L.take((size_t)M * sizeof(int)), orderAt = L.take((size_t)M * sizeof(int));
  const size_t piecesAt = L.take(((size_t)tiles + C) * GP_PV * sizeof(double));
  const size_t camPartAt = L.take((size_t)idivup(C, 32) * GP_CP * sizeof(double));
  const size_t ptPartAt = L.take((size_t)idivup(T, GP_THREADS) * sizeof(double));
  const size_t tempAt = L.take(std::max(scanBytes, sortBytes));
  int r = c.globalpos.grow(L.bytes);
  if (r < 0) return r;
  char *base = c.globalpos.as<char>();

  size_t hBytes = 0;
  const size_t hCamAt = gp_host_layout(C, maxIterations, &hBytes);
  if ((r = c.h_globalpos.grow(hBytes)) < 0) return r;
  GpCam *cams = reinterpret_cast<GpCam *>(c.h_globalpos.as<char>() + hCamAt);
  for (int a = 0; a < C; a++) {
    GpCam &m = cams[a];
    memset(&m, 0, sizeof m);
    for (int i = 0; i < 6; i++) m.K[i] = Ks[9 * (size_t)a + i];
    bool finite = true;
    for (int i = 0; i < 9; i++) finite = finite && std::isfinite(Rs[9 * (size_t)a + i]);
    for (int i = 0; i < 9; i++) m.R[i] = finite ? Rs[9 * (size_t)a + i] : 0.0;
    m.hasR = finite;
    m.pts = static_cast<const SiftPoint *>(sets[a].pts);
    m.n = sets[a].n;
  }

  GpParams prm;
  prm.res = reinterpret_cast<GpResult *>(base + resAt);
  prm.flags = reinterpret_cast<unsigned int *>(base + flagsAt);
  prm.trace = reinterpret_cast<double *>(base + traceAt);
  prm.cams = reinterpret_cast<GpCam *>(base + camAt);
  prm.pts = reinterpret_cast<GpPt *>(base + ptAt);
  prm.cnt = reinterpret_cast<int *>(base + cntAt);
  prm.start = reinterpret_cast<int *>(base + startAt);
  prm.obs = reinterpret_cast<GpObs *>(base + obsAt);
  prm.keys = reinterpret_cast<int *>(base + keysAt);
  prm.vals = reinterpret_cast<int *>(base + valsAt);
  prm.keysS = reinterpret_cast<const int *>(base + keysSAt);
  prm.order = reinterpret_cast<const int *>(base + orderAt);
  prm.pieces = reinterpret_cast<double *>(base + piecesAt);
  prm.camPart = reinterpret_cast<double *>(base + camPartAt);
  prm.ptPart = reinterpret_cast<double *>(base + ptPartAt);
  prm.offsets = offsets;
  prm.members = reinterpret_cast<const int2 *>(members);
  prm.use = use;
  prm.points = points;
  prm.tol2 = linearTol * linearTol;
  prm.c2 = lossScale * lossScale;
  prm.seed = seed;
  prm.numImages = C;
  prm.numTracks = T;
  prm.numMembers = M;
  prm.maxIterations = maxIterations;
  prm.maxLinear = maxLinearIterations;
  prm.loss = loss;
  prm.refImage = refImage;

  const int wave = coop_grid<gp_kernel, GP_THREADS>("cs_global_positioning");
  if (wave < 0) return wave;
  const cudaStream_t st = c.stream;
  CS_CUDA(cudaMemsetAsync(base, 0, zeroEnd, st));
  if (C) CS_CUDA(cudaMemcpyAsync(prm.cams, cams, (size_t)C * sizeof(GpCam), cudaMemcpyHostToDevice, st));
  gp_count_kernel<<<std::max(idivup(T, GP_THREADS), 1), GP_THREADS, 0, st>>>(prm);
  count_launch();
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cub::DeviceScan::ExclusiveSum(base + tempAt, scanBytes, prm.cnt, prm.start, T + 1, st));
  gp_fill_kernel<<<std::max(idivup(std::max(T, M), GP_THREADS), 1), GP_THREADS, 0, st>>>(prm);
  count_launch();
  CS_CUDA(cudaGetLastError());
  if (M > 0)
    CS_CUDA(cub::DeviceRadixSort::SortPairs(base + tempAt, sortBytes, prm.keys, const_cast<int *>(prm.keysS), prm.vals,
                                            const_cast<int *>(prm.order), M, 0, bits, st));
  void *args[] = {&prm};
  CS_CUDA(cudaLaunchCooperativeKernel((const void *)gp_kernel, dim3(wave), dim3(GP_THREADS), args, 0, st));
  count_launch();
  CS_CUDA(cudaMemcpyAsync(c.h_globalpos.p, base + resAt, flagsAt - resAt, cudaMemcpyDeviceToHost, st));
  if (C) CS_CUDA(cudaMemcpyAsync(cams, prm.cams, (size_t)C * sizeof(GpCam), cudaMemcpyDeviceToHost, st));
  return 0;
}

int globalpos_result(const DeviceCtx &c, int numImages, const double *Rs, int maxIterations, double *t_out,
                     double cost[2], double *trace, long long stats[8])
{
  const size_t camAt = gp_host_layout(numImages, maxIterations, nullptr);
  Layout H(256);
  H.take(sizeof(GpResult));
  const size_t trAt = H.take((size_t)maxIterations * 4 * sizeof(double));
  const GpResult *res = c.h_globalpos.as<const GpResult>();
  const GpCam *cams = reinterpret_cast<const GpCam *>(c.h_globalpos.as<const char>() + camAt);
  for (int a = 0; a < numImages; a++) {
    const GpCam &m = cams[a];
    const bool has = m.hasR && m.end > m.start;
    for (int i = 0; i < 3; i++) {
      const double *R = Rs + 9 * (size_t)a + 3 * i;
      t_out[3 * (size_t)a + i] =
          has ? -(R[0] * m.c[0] + R[1] * m.c[1] + R[2] * m.c[2]) / res->scale : NAN;
    }
  }
  cost[0] = res->cost[0];
  cost[1] = res->cost[1];
  if (trace) memcpy(trace, c.h_globalpos.as<const char>() + trAt, (size_t)maxIterations * 4 * sizeof(double));
  if (stats)
    for (int k = 0; k < 8; k++) stats[k] = (long long)res->stats[k];
  return (int)res->accepted;
}

}  // namespace cs
