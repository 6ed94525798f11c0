// pose.cu -- camera registration against known 3-D points (cs_absolute_pose_batch): RANSAC over Lambda Twist P3P
// hypotheses in FP64, scored with triangulation's reprojection inlier rule, then one Levenberg-Marquardt refinement of
// the winner.  The rules are stated in cudasift_b200.h at cs_absolute_pose_batch; tests/pose_oracle.py restates them in
// float64.
//
// Every launch runs a wave of jobs (the host cuts the batch's non-empty jobs into waves whose slot scratch fits 256
// MiB).  Five launches per wave:
//   1. gather  one warp per job: the valid correspondences in feature order, compacted by ballots (pixel, world point,
//              bearing, feature index); NaN / 0 per-feature outputs for the features that are not valid; the job's
//              state reset.
//   2. hyp     one thread per sample, a fixed number of CTAs per job: the three draws of cs_verify_pairs' sampler and
//              the P3P solver, up to 4 poses in the sample's slots (an empty slot holds NaN).
//   3. score   grid (correspondence chunks of all jobs, slot blocks): correspondence tiles in shared memory, one slot
//              per thread, integer counts.  A CTA finds its job with table_find over the host-built chunk bases.
//   4. argmax  packed atomicMax of (count << 32 | ~slot) per job: the most inliers, then the lowest slot.
//   5. refine  one warp per job: Levenberg-Marquardt over the winner's inliers.  Lanes take ranks lane, lane + 32, ...
//              and fixed xor butterflies combine the 28 sums, so every lane holds the same bits and runs the same 6x6
//              Cholesky; then the keep rule, the pose, the count, the statistics and the per-feature outputs.
// Nothing depends on scheduling or on the other jobs of a wave: counts are integer sums, the winner an integer max,
// and every floating-point sum of a job runs in an order fixed by its own correspondences.
#include <algorithm>
#include <cmath>
#include <vector>
#include <math_constants.h>

#include "common.cuh"
#include "vp_math.cuh"

namespace cs {

namespace {

constexpr int PS_SLOTS = 4;          // poses per sample
constexpr int PS_SLOT_DOUBLES = 12;  // R row-major, then t
constexpr int PS_HYP_T = 128;        // samples per hypothesis CTA
constexpr int PS_SC_T = 128;         // slots per scoring CTA
constexpr int PS_CHUNK = 1024;       // correspondences per scoring CTA
constexpr int PS_TILE = 256;         // correspondences per shared-memory tile
constexpr int PS_WARPS = 4;          // jobs per CTA of the gather and refine kernels
constexpr double PS_EPS = 1e-10;     // degeneracy thresholds: collinear world points, near-parallel bearings
constexpr int PS_GN_STEPS = 5;
constexpr int PS_LM_ITERS = 20;
constexpr double PS_LM_LAMBDA0 = 1e-3, PS_LM_STEP_TOL = 1e-12, PS_LM_COST_TOL = 1e-12;

// A valid correspondence: its world point, bearing, pixel and feature index.
struct PoseCorr {
  double X[3], b[3];
  float x, y;
  int pos, pad;
};

// One job as the kernels read it.
struct PoseJobDev {
  const SiftPoint *pts;
  const int *pointOf;
  float *errors;
  unsigned char *inlier;
  unsigned long long seed;
  double K[6];                      // K[0..5] (upper-triangular, K[3] = 0)
  int n;
  int corrBase;                     // its first correspondence in the wave's scratch
  int scoreBase;                    // its first scoring CTA
  int pad;
};

// A job's state: written by the kernels, copied back after the wave.
struct PoseState {
  double R[9], t[3];
  unsigned long long best;          // packed arg-max key; 0 = no pose scored
  unsigned long long samples;       // non-degenerate samples
  unsigned long long poses;         // live slots
  long long stats[8];
  int V, invalid, count, pad;
};

struct PoseWave {
  const PoseJobDev *jobs;
  int numJobs, numLoops;
  PoseCorr *corr;
  double *slots;                    // [job][4 numLoops][12]
  unsigned int *slotCounts;         // [job][4 numLoops]
  PoseState *st;
  const double *points;
  int numPoints;
  double thr2;
};

// ---- shared math (host and device: the solver can be exercised on a CPU build) -------------------------------------
__host__ __device__ inline double ps_dot(const double *u, const double *v) { return u[0] * v[0] + u[1] * v[1] + u[2] * v[2]; }
__host__ __device__ inline void ps_cross(const double *u, const double *v, double *w)
{
  w[0] = u[1] * v[2] - u[2] * v[1];
  w[1] = u[2] * v[0] - u[0] * v[2];
  w[2] = u[0] * v[1] - u[1] * v[0];
}

// The largest real root of g^3 + b g^2 + c g + d: the closed form (Cardano when the discriminant is >= 0, else the
// trigonometric form), then two Newton steps, each taken when the derivative is nonzero and the result finite.
__host__ __device__ inline double ps_cubic_root(double b, double c, double d)
{
  const double p = c - b * b / 3.0, q = 2.0 * b * b * b / 27.0 - b * c / 3.0 + d;
  const double disc = 0.25 * q * q + p * p * p / 27.0;
  double z;
  if (disc >= 0.0) {
    const double s = sqrt(disc);
    z = cbrt(-0.5 * q + s) + cbrt(-0.5 * q - s);
  } else {
    const double r = sqrt(-p / 3.0);
    z = 2.0 * r * cos(acos(fmin(1.0, fmax(-1.0, -0.5 * q / (r * r * r)))) / 3.0);
  }
  double g = z - b / 3.0;
  for (int it = 0; it < 2; it++) {
    const double f = ((g + b) * g + c) * g + d, fp = (3.0 * g + 2.0 * b) * g + c;
    if (fp == 0.0) break;
    const double g1 = g - f / fp;
    if (isfinite(g1)) g = g1;
  }
  return g;
}

// Up to 5 Newton steps on the three distance equations r_ij = li^2 + lj^2 + bij li lj - aij; a step is kept only when
// it is finite and lowers |r1| + |r2| + |r3|, else the refinement stops.
__host__ __device__ inline void ps_refine_depths(double *L, double a12, double a13, double a23, double b12, double b13,
                                                 double b23)
{
  for (int it = 0; it < PS_GN_STEPS; it++) {
    const double l1 = L[0], l2 = L[1], l3 = L[2];
    const double r1 = l1 * l1 + l2 * l2 + b12 * l1 * l2 - a12, r2 = l1 * l1 + l3 * l3 + b13 * l1 * l3 - a13,
                 r3 = l2 * l2 + l3 * l3 + b23 * l2 * l3 - a23;
    const double e = fabs(r1) + fabs(r2) + fabs(r3);
    if (e == 0.0) break;
    const double v0 = 2.0 * l1 + b12 * l2, v1 = 2.0 * l2 + b12 * l1, v3 = 2.0 * l1 + b13 * l3, v5 = 2.0 * l3 + b13 * l1,
                 v7 = 2.0 * l2 + b23 * l3, v8 = 2.0 * l3 + b23 * l2;
    const double det = -v0 * v5 * v7 - v1 * v3 * v8;
    if (det == 0.0) break;
    const double inv = 1.0 / det;
    const double n1 = l1 - (-v5 * v7 * r1 - v1 * v8 * r2 + v1 * v5 * r3) * inv;
    const double n2 = l2 - (-v3 * v8 * r1 + v0 * v8 * r2 - v0 * v5 * r3) * inv;
    const double n3 = l3 - (v3 * v7 * r1 - v0 * v7 * r2 - v1 * v3 * r3) * inv;
    if (!isfinite(n1) || !isfinite(n2) || !isfinite(n3)) break;
    const double s1 = n1 * n1 + n2 * n2 + b12 * n1 * n2 - a12, s2 = n1 * n1 + n3 * n3 + b13 * n1 * n3 - a13,
                 s3 = n2 * n2 + n3 * n3 + b23 * n2 * n3 - a23;
    if (!(fabs(s1) + fabs(s2) + fabs(s3) < e)) break;
    L[0] = n1; L[1] = n2; L[2] = n3;
  }
}

// Lambda Twist P3P (Persson & Nordberg, ECCV 2018) on bearings y[k] and world points X[k] in draw order.  Writes up to
// 4 poses (R row-major, then t) to out in slot order and returns their number; -1 for a degenerate sample.  Every
// choice is stated at cs_absolute_pose_batch in cudasift_b200.h.
__host__ __device__ inline int ps_p3p(const double (&y)[3][3], const double (&X)[3][3], double (&out)[PS_SLOTS][12])
{
  double d12[3], d13[3], d23[3], nn[3];
  for (int i = 0; i < 3; i++) { d12[i] = X[0][i] - X[1][i]; d13[i] = X[0][i] - X[2][i]; d23[i] = X[1][i] - X[2][i]; }
  const double a12 = ps_dot(d12, d12), a13 = ps_dot(d13, d13), a23 = ps_dot(d23, d23);
  ps_cross(d12, d13, nn);
  if (!(ps_dot(nn, nn) > PS_EPS * a12 * a13)) return -1;
  const double c12 = ps_dot(y[0], y[1]), c13 = ps_dot(y[0], y[2]), c23 = ps_dot(y[1], y[2]);
  const double s12 = 1.0 - c12 * c12, s13 = 1.0 - c13 * c13, s23 = 1.0 - c23 * c23;
  if (!(s12 > PS_EPS && s13 > PS_EPS && s23 > PS_EPS)) return -1;
  const double b12 = -2.0 * c12, b13 = -2.0 * c13, b23 = -2.0 * c23;
  const double blob = c12 * c23 * c13 - 1.0;
  const double p3 = a13 * (a23 * s13 - a13 * s23);
  const double p2 = 2.0 * blob * a23 * a13 + a13 * (2.0 * a12 + a13) * s23 + a23 * (a23 - a12) * s13;
  const double p1 = a23 * (a13 - a23) * s12 - a12 * a12 * s23 - 2.0 * a12 * (blob * a23 + a13 * s23);
  const double p0 = a12 * (a12 * s23 - a23 * s12);
  if (p3 == 0.0) return -1;
  const double g = ps_cubic_root(p2 / p3, p1 / p3, p0 / p3);
  // D0 = D1 - g D2, rank 2 at a root: its two eigenvalues of largest magnitude by vp_jacobi<3>
  double A[3][3], V[3][3];
  A[0][0] = a23 * (1.0 - g);
  A[0][1] = A[1][0] = 0.5 * a23 * b12;
  A[0][2] = A[2][0] = -0.5 * a23 * b13 * g;
  A[1][1] = a23 - a12 + a13 * g;
  A[1][2] = A[2][1] = 0.5 * b23 * (a13 * g - a12);
  A[2][2] = g * (a13 - a23) - a12;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      if (!isfinite(A[i][j])) return -1;
  vp_jacobi<3>(A, V);
  // the order of |eigenvalue| descending, the lower index first on ties
  int o0 = 0, o1 = 1, o2 = 2, t;
  if (fabs(A[o1][o1]) > fabs(A[o0][o0])) { t = o0; o0 = o1; o1 = t; }
  if (fabs(A[o2][o2]) > fabs(A[o1][o1])) { t = o1; o1 = o2; o2 = t; }
  if (fabs(A[o1][o1]) > fabs(A[o0][o0]) || (fabs(A[o1][o1]) == fabs(A[o0][o0]) && o1 < o0)) { t = o0; o0 = o1; o1 = t; }
  const double e0 = A[o0][o0], e1 = A[o1][o1];
  if (e0 == 0.0) return -1;
  const double v = sqrt(fmax(0.0, -e1 / e0));
  double Ls[4][3];
  int nl = 0;
  for (int br = 0; br < 2; br++) {
    const double s = br ? -v : v;
    const double w2 = 1.0 / (s * V[0][o1] - V[0][o0]);
    const double w0 = (V[1][o0] - s * V[1][o1]) * w2, w1 = (V[2][o0] - s * V[2][o1]) * w2;
    const double qa = 1.0 / ((a13 - a12) * w1 * w1 - a12 * b13 * w1 - a12);
    const double qb = (a13 * b12 * w1 - a12 * b13 * w0 - 2.0 * w0 * w1 * (a12 - a13)) * qa;
    const double qc = ((a13 - a12) * w0 * w0 + a13 * b12 * w0 + a13) * qa;
    const double disc = qb * qb - 4.0 * qc;
    if (!(disc >= 0.0)) continue;
    const double sq = sqrt(disc);
    const double tau1 = qb < 0.0 ? 0.5 * (-qb + sq) : 0.5 * (-qb - sq);
    const double tau2 = tau1 != 0.0 ? qc / tau1 : 0.0;          // tau1 == 0: no second root (0 is not > 0)
    for (int k = 0; k < 2; k++) {
      const double tau = k ? tau2 : tau1;
      if (!(tau > 0.0)) continue;
      const double dd = a23 / (tau * (b23 + tau) + 1.0);
      if (!(dd > 0.0)) continue;
      const double l2 = sqrt(dd), l3 = tau * l2, l1 = w0 * l2 + w1 * l3;
      if (l1 > 0.0) { Ls[nl][0] = l1; Ls[nl][1] = l2; Ls[nl][2] = l3; nl++; }
    }
  }
  // the inverse of the world frame [d12 d13 n]: rows (d13 x n, n x d12, d12 x d13) / det
  double inv[3][3];
  ps_cross(d13, nn, inv[0]);
  ps_cross(nn, d12, inv[1]);
  ps_cross(d12, d13, inv[2]);
  const double det = ps_dot(d12, inv[0]);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) inv[i][j] = inv[i][j] / det;
  int r = 0;
  for (int k = 0; k < nl; k++) {
    double L[3] = {Ls[k][0], Ls[k][1], Ls[k][2]};
    ps_refine_depths(L, a12, a13, a23, b12, b13, b23);
    if (!(L[0] > 0.0 && L[1] > 0.0 && L[2] > 0.0 && isfinite(L[0]) && isfinite(L[1]) && isfinite(L[2]))) continue;
    double r0[3], yd1[3], yd2[3], yd3[3];
    for (int i = 0; i < 3; i++) {
      r0[i] = L[0] * y[0][i];
      yd1[i] = r0[i] - L[1] * y[1][i];
      yd2[i] = r0[i] - L[2] * y[2][i];
    }
    ps_cross(yd1, yd2, yd3);
    double *o = out[r];
    bool fin = true;
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) {
        o[3 * i + j] = yd1[i] * inv[0][j] + yd2[i] * inv[1][j] + yd3[i] * inv[2][j];
      }
    for (int i = 0; i < 3; i++) o[9 + i] = r0[i] - (o[3 * i] * X[0][0] + o[3 * i + 1] * X[0][1] + o[3 * i + 2] * X[0][2]);
    for (int i = 0; i < 12; i++) fin = fin && isfinite(o[i]);
    if (fin) r++;
  }
  return r;
}

// P = K [R | t] (row-major 3 x 4) with an explicit fma chain, so that every kernel builds the same bits.
__device__ __forceinline__ void ps_camera(const double *K, const double *R, const double *t, double (&P)[12])
{
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const double c0 = j < 3 ? R[j] : t[0], c1 = j < 3 ? R[3 + j] : t[1], c2 = j < 3 ? R[6 + j] : t[2];
    P[j] = fma(K[0], c0, fma(K[1], c1, K[2] * c2));
    P[4 + j] = fma(K[4], c1, K[5] * c2);
    P[8 + j] = c2;
  }
}

// ---- kernels --------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(PS_WARPS * 32) pose_gather_kernel(PoseWave w)
{
  const int lane = threadIdx.x & 31, j = blockIdx.x * PS_WARPS + (threadIdx.x >> 5);
  if (j >= w.numJobs) return;
  const PoseJobDev &job = w.jobs[j];
  PoseCorr *corr = w.corr + job.corrBase;
  int V = 0, invalid = 0;
  for (int b0 = 0; b0 < job.n; b0 += 32) {
    const int f = b0 + lane;
    bool ok = false;
    PoseCorr c;
    if (f < job.n) {
      const int p = job.pointOf[f];
      if (p >= 0) {
        if (p < w.numPoints) {
          for (int i = 0; i < 3; i++) c.X[i] = w.points[3 * (size_t)p + i];
          c.x = job.pts[f].xpos;
          c.y = job.pts[f].ypos;
          ok = isfinite(c.X[0]) && isfinite(c.X[1]) && isfinite(c.X[2]) && isfinite(c.x) && isfinite(c.y);
        }
        invalid += !ok;
      }
      if (!ok) {
        if (job.errors) job.errors[f] = CUDART_NAN_F;
        if (job.inlier) job.inlier[f] = 0;
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    if (ok) {
      double cx, cy;
      vp_calibrate(job.K, (double)c.x, (double)c.y, cx, cy);
      const double nrm = sqrt(cx * cx + cy * cy + 1.0);
      c.b[0] = cx / nrm; c.b[1] = cy / nrm; c.b[2] = 1.0 / nrm;
      c.pos = f;
      c.pad = 0;
      corr[V + __popc(bal & ((1u << lane) - 1u))] = c;
    }
    V += __popc(bal);
  }
  invalid = __reduce_add_sync(0xffffffffu, invalid);
  if (lane == 0) {
    PoseState &s = w.st[j];
    s.V = V;
    s.invalid = invalid;
    s.best = 0;
    s.samples = 0;
    s.poses = 0;
  }
}

__global__ void __launch_bounds__(PS_HYP_T) pose_hyp_kernel(PoseWave w)
{
  int j, smp;
  double *slot;
  if (!vp_hyp_sample<PS_HYP_T, PS_SLOTS, PS_SLOT_DOUBLES>(w.numLoops, w.slots, w.slotCounts, j, smp, slot)) return;
  const PoseJobDev &job = w.jobs[j];
  int idx[3];
  if (!vp_draw<3>(job.seed, smp, w.st[j].V, idx)) return;
  const PoseCorr *corr = w.corr + job.corrBase;
  double y[3][3], X[3][3], out[PS_SLOTS][12];
  for (int k = 0; k < 3; k++)
    for (int i = 0; i < 3; i++) { y[k][i] = corr[idx[k]].b[i]; X[k][i] = corr[idx[k]].X[i]; }
  const int np = ps_p3p(y, X, out);
  if (np < 0) return;
  atomicAdd(&w.st[j].samples, 1ull);
  for (int r = 0; r < np; r++)
    for (int i = 0; i < PS_SLOT_DOUBLES; i++) slot[PS_SLOT_DOUBLES * r + i] = out[r][i];
}

struct PoseTileEntry {
  double X[3];
  float x, y;
};

__global__ void __launch_bounds__(PS_SC_T) pose_score_kernel(PoseWave w)
{
  __shared__ PoseTileEntry s_c[PS_TILE];
  const int j = table_find(w.jobs, w.numJobs, &PoseJobDev::scoreBase, (int)blockIdx.x);
  const PoseJobDev &job = w.jobs[j];
  const int V = w.st[j].V;
  const int c0 = ((int)blockIdx.x - job.scoreBase) * PS_CHUNK;
  if (c0 >= V) return;
  const int c1 = min(V, c0 + PS_CHUNK);
  const int S = PS_SLOTS * w.numLoops, slot = blockIdx.y * PS_SC_T + threadIdx.x;
  const double *m = w.slots + ((size_t)j * S + slot) * PS_SLOT_DOUBLES;
  const bool live = slot < S && !isnan(m[0]);
  double P[12];
  if (live) ps_camera(job.K, m, m + 9, P);
  const PoseCorr *corr = w.corr + job.corrBase;
  unsigned int cnt = 0;
  for (int t0 = c0; t0 < c1; t0 += PS_TILE) {
    const int tn = min(PS_TILE, c1 - t0);
    __syncthreads();
    for (int k = threadIdx.x; k < tn; k += PS_SC_T) {
      const PoseCorr &c = corr[t0 + k];
      s_c[k].X[0] = c.X[0]; s_c[k].X[1] = c.X[1]; s_c[k].X[2] = c.X[2];
      s_c[k].x = c.x; s_c[k].y = c.y;
    }
    __syncthreads();
    if (live)
      for (int k = 0; k < tn; k++) {
        const double X[3] = {s_c[k].X[0], s_c[k].X[1], s_c[k].X[2]};
        cnt += tr_inlier(P, X, s_c[k].x, s_c[k].y, w.thr2);
      }
  }
  if (live && cnt) atomicAdd(&w.slotCounts[(size_t)j * S + slot], cnt);
}

// idivup(slots, 256) CTAs per job, so that no warp holds two jobs' slots
__global__ void __launch_bounds__(256) pose_argmax_kernel(PoseWave w)
{
  const int S = PS_SLOTS * w.numLoops, per = (S + 255) / 256, j = blockIdx.x / per;
  const int slot = (blockIdx.x - j * per) * 256 + threadIdx.x;
  const bool live = slot < S && !isnan(w.slots[((size_t)j * S + slot) * PS_SLOT_DOUBLES]);
  vp_argmax_warp(live, w.slotCounts + (size_t)j * S + slot, slot, &w.st[j].best, &w.st[j].poses);
}

constexpr int PS_SUMS = 28;          // H (21, upper triangle row by row), g (6), the cost

// This lane's share of the refinement sums at pose (R, t) over the winner's inliers (Pw) among ranks lane, lane + 32,
// ..., then the xor butterfly (every lane ends with the same bits).  Returns whether every depth is > 0.
__device__ bool ps_lm_terms(const PoseCorr *corr, int V, const double *K, const double (&Pw)[12], double thr2,
                            const double (&R)[9], const double (&t)[3], double (&s)[PS_SUMS])
{
  const int lane = threadIdx.x & 31;
  for (int i = 0; i < PS_SUMS; i++) s[i] = 0.0;
  bool front = true;
  for (int r = lane; r < V; r += 32) {
    const PoseCorr &c = corr[r];
    const double X[3] = {c.X[0], c.X[1], c.X[2]};
    if (!tr_inlier(Pw, X, c.x, c.y, thr2)) continue;
    double Xc[3];
    for (int i = 0; i < 3; i++) Xc[i] = R[3 * i] * X[0] + R[3 * i + 1] * X[1] + R[3 * i + 2] * X[2] + t[i];
    const double z = Xc[2];
    front = front && z > 0.0;
    const double a = Xc[0] / z, b = Xc[1] / z;
    const double res[2] = {K[0] * a + K[1] * b + K[2] - (double)c.x, K[4] * b + K[5] - (double)c.y};
    const double gr[2][3] = {{K[0] / z, K[1] / z, -(K[0] * a + K[1] * b) / z}, {0.0, K[4] / z, -K[4] * b / z}};
    for (int q = 0; q < 2; q++) {
      double J[6];
      ps_cross(Xc, gr[q], J);
      J[3] = gr[q][0]; J[4] = gr[q][1]; J[5] = gr[q][2];
      int k = 0;
      for (int i = 0; i < 6; i++)
        for (int m = i; m < 6; m++) s[k++] += J[i] * J[m];
      for (int i = 0; i < 6; i++) s[21 + i] += J[i] * res[q];
      s[27] += res[q] * res[q];
    }
  }
  vp_warp_sum(s);
  return __all_sync(0xffffffffu, front);
}

// (H + lam diag(H)) x = -g by Cholesky; false when a pivot is not > 0 or not finite
__device__ bool ps_lm_solve(const double (&s)[PS_SUMS], double lam, double (&x)[6])
{
  double M[6][6], L[6][6];
  int k = 0;
  for (int i = 0; i < 6; i++)
    for (int m = i; m < 6; m++) { M[i][m] = M[m][i] = s[k]; k++; }
  for (int i = 0; i < 6; i++) M[i][i] += lam * M[i][i];
  for (int jj = 0; jj < 6; jj++) {
    double d = M[jj][jj];
    for (int q = 0; q < jj; q++) d -= L[jj][q] * L[jj][q];
    if (!(d > 0.0) || !isfinite(d)) return false;
    L[jj][jj] = sqrt(d);
    for (int i = jj + 1; i < 6; i++) {
      double e = M[i][jj];
      for (int q = 0; q < jj; q++) e -= L[i][q] * L[jj][q];
      L[i][jj] = e / L[jj][jj];
    }
  }
  double z[6];
  for (int i = 0; i < 6; i++) {
    double e = -s[21 + i];
    for (int q = 0; q < i; q++) e -= L[i][q] * z[q];
    z[i] = e / L[i][i];
  }
  for (int i = 5; i >= 0; i--) {
    double e = z[i];
    for (int q = i + 1; q < 6; q++) e -= L[q][i] * x[q];
    x[i] = e / L[i][i];
  }
  return true;
}

// R' = exp([w]x) R, t' = exp([w]x) t + delta (vp_rotate)
__device__ void ps_update(const double (&R)[9], const double (&t)[3], const double (&x)[6], double (&R1)[9],
                          double (&t1)[3])
{
  double Q[9];
  vp_rotate(x, R, R1, Q);
  for (int i = 0; i < 3; i++) t1[i] = Q[3 * i] * t[0] + Q[3 * i + 1] * t[1] + Q[3 * i + 2] * t[2] + x[3 + i];
}

__device__ int ps_count(const PoseCorr *corr, int V, const double (&P)[12], double thr2)
{
  int cnt = 0;
  for (int r = (int)(threadIdx.x & 31); r < V; r += 32) {
    const double X[3] = {corr[r].X[0], corr[r].X[1], corr[r].X[2]};
    cnt += tr_inlier(P, X, corr[r].x, corr[r].y, thr2);
  }
  return __reduce_add_sync(0xffffffffu, cnt);
}

__global__ void __launch_bounds__(PS_WARPS * 32) pose_refine_kernel(PoseWave w)
{
  const int lane = threadIdx.x & 31, j = blockIdx.x * PS_WARPS + (threadIdx.x >> 5);
  if (j >= w.numJobs) return;
  const PoseJobDev &job = w.jobs[j];
  PoseState &st = w.st[j];
  const PoseCorr *corr = w.corr + job.corrBase;
  const int V = st.V, S = PS_SLOTS * w.numLoops;
  const unsigned long long best = st.best;
  int slot = -1, count0 = 0, count = 0, kept = 0;
  double R[9], t[3];
  if (best) {
    slot = (int)~(unsigned int)best;
    count0 = (int)(best >> 32);
    const double *m = w.slots + ((size_t)j * S + slot) * PS_SLOT_DOUBLES;
    for (int i = 0; i < 9; i++) R[i] = m[i];
    for (int i = 0; i < 3; i++) t[i] = m[9 + i];
    count = count0;
  }
  if (best && count0 >= 3) {
    double Pw[12];
    ps_camera(job.K, R, t, Pw);
    double Rc[9], tc[3], s[PS_SUMS];
    for (int i = 0; i < 9; i++) Rc[i] = R[i];
    for (int i = 0; i < 3; i++) tc[i] = t[i];
    ps_lm_terms(corr, V, job.K, Pw, w.thr2, Rc, tc, s);
    double lam = PS_LM_LAMBDA0;
    for (int it = 0; it < PS_LM_ITERS; it++) {
      double x[6];
      if (!ps_lm_solve(s, lam, x)) { lam *= 10.0; continue; }
      double R1[9], t1[3], s1[PS_SUMS];
      ps_update(Rc, tc, x, R1, t1);
      const bool front = ps_lm_terms(corr, V, job.K, Pw, w.thr2, R1, t1, s1);
      if (front && s1[27] < s[27]) {
        const double dec = s[27] - s1[27];
        double big = 0.0;
        for (int i = 0; i < 6; i++) big = fmax(big, fabs(x[i]));
        const bool stop = big <= PS_LM_STEP_TOL || dec <= PS_LM_COST_TOL * s[27];
        for (int i = 0; i < 9; i++) Rc[i] = R1[i];
        for (int i = 0; i < 3; i++) tc[i] = t1[i];
        for (int i = 0; i < PS_SUMS; i++) s[i] = s1[i];
        lam /= 10.0;
        if (stop) break;
      } else {
        lam *= 10.0;
      }
    }
    bool fin = true;
    for (int i = 0; i < 9; i++) fin = fin && isfinite(Rc[i]);
    for (int i = 0; i < 3; i++) fin = fin && isfinite(tc[i]);
    if (fin) {
      double P1[12];
      ps_camera(job.K, Rc, tc, P1);
      const int c1 = ps_count(corr, V, P1, w.thr2);
      if (c1 >= count0) {
        kept = 1;
        count = c1;
        for (int i = 0; i < 9; i++) R[i] = Rc[i];
        for (int i = 0; i < 3; i++) t[i] = tc[i];
      }
    }
  }
  const bool has = best && count >= 3;
  if (lane == 0) {
    for (int i = 0; i < 9; i++) st.R[i] = has ? R[i] : 0.0;
    for (int i = 0; i < 3; i++) st.t[i] = has ? t[i] : 0.0;
    st.count = has ? count : 0;
    st.stats[0] = V;
    st.stats[1] = st.invalid;
    st.stats[2] = (long long)st.samples;
    st.stats[3] = (long long)st.poses;
    st.stats[4] = slot;
    st.stats[5] = count0;
    st.stats[6] = kept;
    st.stats[7] = has ? count : 0;
  }
  if (job.errors || job.inlier) {
    double P[12];
    if (has) ps_camera(job.K, R, t, P);
    for (int r = lane; r < V; r += 32) {
      const PoseCorr &c = corr[r];
      float err = CUDART_NAN_F;
      unsigned char in = 0;
      if (has) {
        const double X[3] = {c.X[0], c.X[1], c.X[2]};
        tr_reproject(P, X, c.x, c.y, w.thr2, err, in);
      }
      if (job.errors) job.errors[c.pos] = err;
      if (job.inlier) job.inlier[c.pos] = in;
    }
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------
// The waves of a batch, a job's extent being its correspondence count.
WavePlan pose_plan(const cs_pose_job *jobs, int numJobs, int numLoops)
{
  const size_t slotBytes = (size_t)PS_SLOTS * numLoops * (PS_SLOT_DOUBLES * sizeof(double) + sizeof(unsigned int));
  return wave_plan(jobs, numJobs, slotBytes, [](const cs_pose_job &a) { return (size_t)a.n; });
}

struct PoseLayout {
  size_t jobs, corr, slots, slotCounts, state, bytes;
};

// The device table of the batch's non-empty jobs, then the scratch of one wave (reused by the next).
PoseLayout pose_layout(const WavePlan &p, int numLoops)
{
  PoseLayout L;
  Layout o(256);
  const size_t live = std::max(p.live.size(), (size_t)1), J = std::min(live, (size_t)p.perWave);
  const size_t S = (size_t)PS_SLOTS * numLoops * J;
  L.jobs = o.take(live * sizeof(PoseJobDev));
  L.corr = o.take(std::max(p.extent, (size_t)1) * sizeof(PoseCorr));
  L.slots = o.take(S * PS_SLOT_DOUBLES * sizeof(double));
  L.slotCounts = o.take(S * sizeof(unsigned int));
  L.state = o.take(J * sizeof(PoseState));
  L.bytes = o.bytes;
  return L;
}

}  // namespace

int pose_enqueue(DeviceCtx &c, const double *points, int numPoints, const cs_pose_job *jobs, int numJobs,
                 const double *Ks, int numLoops, double maxError, bool full)
{
  const WavePlan plan = pose_plan(jobs, numJobs, numLoops);
  const int live = (int)plan.live.size();
  if (live == 0) return 0;
  const PoseLayout L = pose_layout(plan, numLoops);
  int r;
  if ((r = c.pose.grow(L.bytes)) < 0) return r;
  PoseState *h_states;
  PoseJobDev *h_jobs;
  if ((r = pinned_states_and_jobs(c.h_pose, live, h_states, h_jobs)) < 0) return r;
  char *b = c.pose.as<char>();
  // the table; the correspondence and score bases count from the first job of each wave
  int corrBase = 0, scoreBase = 0;
  for (int q = 0; q < live; q++) {
    if (q % plan.perWave == 0) corrBase = scoreBase = 0;
    const int p = plan.live[q];
    const cs_pose_job &a = jobs[p];
    PoseJobDev &t = h_jobs[q];
    t.pts = static_cast<const SiftPoint *>(a.pts);
    t.pointOf = a.pointOf;
    t.errors = a.errors;
    t.inlier = a.inlier;
    t.seed = a.seed;
    for (int i = 0; i < 6; i++) t.K[i] = Ks[9 * (size_t)p + i];
    t.n = a.n;
    t.corrBase = corrBase;
    t.scoreBase = scoreBase;
    t.pad = 0;
    corrBase += a.n;
    scoreBase += idivup(a.n, PS_CHUNK);
  }
  PoseJobDev *d_jobs = reinterpret_cast<PoseJobDev *>(b + L.jobs);
  const cudaStream_t st = c.stream;
  CS_CUDA(cudaMemcpyAsync(d_jobs, h_jobs, (size_t)live * sizeof(PoseJobDev), cudaMemcpyHostToDevice, st));
  PoseWave w;
  w.numLoops = numLoops;
  w.corr = reinterpret_cast<PoseCorr *>(b + L.corr);
  w.slots = reinterpret_cast<double *>(b + L.slots);
  w.slotCounts = reinterpret_cast<unsigned int *>(b + L.slotCounts);
  w.st = reinterpret_cast<PoseState *>(b + L.state);
  w.points = points;
  w.numPoints = numPoints;
  w.thr2 = maxError * maxError;
  const int S = PS_SLOTS * numLoops;
  const int hypPerJob = idivup(numLoops, PS_HYP_T), argPerJob = idivup(S, 256), slotBlocks = idivup(S, PS_SC_T);
  cudaEvent_t *tev = full ? match_timing_events() : nullptr;
  for (int q0 = 0; q0 < live; q0 += plan.perWave) {
    const int nj = std::min(plan.perWave, live - q0);
    const PoseJobDev &last = h_jobs[q0 + nj - 1];
    const int chunks = last.scoreBase + idivup(last.n, PS_CHUNK);
    w.jobs = d_jobs + q0;
    w.numJobs = nj;
    if (tev) cudaEventRecord(tev[0], st);
    pose_gather_kernel<<<idivup(nj, PS_WARPS), PS_WARPS * 32, 0, st>>>(w);
    if (tev) cudaEventRecord(tev[1], st);
    pose_hyp_kernel<<<nj * hypPerJob, PS_HYP_T, 0, st>>>(w);
    if (tev) cudaEventRecord(tev[2], st);
    pose_score_kernel<<<dim3(chunks, slotBlocks), PS_SC_T, 0, st>>>(w);
    count_launch(3);
    if (full) {
      if (tev) cudaEventRecord(tev[3], st);
      pose_argmax_kernel<<<nj * argPerJob, 256, 0, st>>>(w);
      if (tev) cudaEventRecord(tev[4], st);
      pose_refine_kernel<<<idivup(nj, PS_WARPS), PS_WARPS * 32, 0, st>>>(w);
      if (tev) cudaEventRecord(tev[5], st);
      count_launch(2);
    }
    CS_CUDA(cudaGetLastError());
    CS_CUDA(cudaMemcpyAsync(h_states + q0, w.st, (size_t)nj * sizeof(PoseState), cudaMemcpyDeviceToHost, st));
    if (tev) {
      static const char *const stages[] = {"gather", "hyp", "score", "argmax", "refine"};
      long long n = 0;
      for (int q = q0; q < q0 + nj; q++) n += h_jobs[q].n;
      report_stage_times(tev, stages, 5, "pose timing jobs=%d features=%lld loops=%d", nj, n, numLoops);
    }
  }
  return 0;
}

int pose_result(const DeviceCtx &c, int q, double R[9], double t[3], long long stats[8])
{
  const PoseState *s = c.h_pose.as<const PoseState>() + q;
  for (int i = 0; i < 9; i++) R[i] = s->R[i];
  for (int i = 0; i < 3; i++) t[i] = s->t[i];
  for (int i = 0; i < 8; i++) stats[i] = s->stats[i];
  return s->count;
}

int pose_models_to_host(DeviceCtx &c, const cs_pose_job &job, int numLoops, double *h_R, double *h_t, int *h_counts)
{
  const PoseLayout L = pose_layout(pose_plan(&job, 1, numLoops), numLoops);
  const char *b = c.pose.as<const char>();
  const size_t S = (size_t)PS_SLOTS * numLoops;
  std::vector<double> slots(S * PS_SLOT_DOUBLES);
  CS_CUDA(cudaMemcpyAsync(slots.data(), b + L.slots, slots.size() * sizeof(double), cudaMemcpyDeviceToHost, c.stream));
  CS_CUDA(cudaMemcpyAsync(h_counts, b + L.slotCounts, S * sizeof(int), cudaMemcpyDeviceToHost, c.stream));
  CS_CUDA(cudaStreamSynchronize(c.stream));
  for (size_t k = 0; k < S; k++) {
    const double *m = slots.data() + PS_SLOT_DOUBLES * k;
    const bool empty = std::isnan(m[0]);
    for (int i = 0; i < 9; i++) h_R[9 * k + i] = empty ? NAN : m[i];
    for (int i = 0; i < 3; i++) h_t[3 * k + i] = empty ? NAN : m[9 + i];
  }
  return c.h_pose.as<const PoseState>()->V;
}

}  // namespace cs
