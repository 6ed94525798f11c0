// bundle.cu -- bundle adjustment of cameras and track points (cs_bundle_adjust, cs_bundle_adjust_intrinsics) and the
// undistortion of records (cs_undistort_records).  The rules (used observations, gauge, camera model, residual, loss,
// Levenberg-Marquardt, the Schur-complement solve, the outputs and the summation orders) are stated in cudasift_b200.h
// at cs_bundle_adjust and cs_bundle_adjust_intrinsics; tests/bundle_oracle.py and tests/bundle_intrinsics_oracle.py
// restate them in float64.
//
// Three counted launches, whatever the sizes and iteration counts:
//   1. bundle_count_kernel: per track, its used observations (0 when fewer than 2) and the integer statistics
//   2. (cub scan of the counts: each participating track's first observation)
//      bundle_fill_kernel: the used observations in track order, then member order, and a key (image) per observation
//   3. (cub stable radix sort of (image, observation): every camera's observations in observation order)
//      bundle_kernel: one cooperative launch runs the whole LM loop, phases separated by grid barriers
// The kernels are instantiated per camera block size NC: 6 (w, delta) when no image refines an intrinsic and every
// distortion coefficient is 0, else 9 (w, delta, f, k1, k2); bundle_kernel also per loss (trivial, or robust with
// soft-L1 or Cauchy chosen at run time).  Every NC-sized piece below is a template of NC, so the <6, false>
// instantiation is the kernel of the squared pixel loss with K held.
// Every floating-point sum has a fixed order that depends on the data only (coop.cuh): per point, a thread sums its
// observations in observation order; per camera, the pieces of the sorted observations' tiles; totals over tiles of 256
// tracks (the cost) or 32 cameras (the CG dot products).  No floating-point atomics.  Every branch around a grid barrier
// (the CG stop, the accept, the LM stop) is taken on values that every CTA computes from the same words, written before
// the barrier, by the same instructions in the same order, so every CTA takes the same path; every loop is bounded by
// maxIterations or maxLinearIterations.
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

constexpr int BA_THREADS = 256;
constexpr int BA_WARPS = BA_THREADS / 32;
// Slots per camera tile partial.  p.S p has a slot of its own: CG phase G writes r.r and r.z with no grid barrier after
// the totals of p.S p are read, so they may not share a slot.
constexpr int BA_CP = 3;

// The sizes that grow with the camera block of NC parameters.
template <int NC>
struct BaSize {
  static constexpr int NU = NC * (NC + 1) / 2;   // a packed symmetric NC x NC block
  static constexpr int JD = 2 * NC + 8;          // doubles per observation: J_c (2 x NC), J_p (2 x 3), r (2)
  static constexpr int PV = 2 * NU + 2 * NC;     // a camera piece: U (NU), g (NC), W V*^-1 g_p (NC), the Schur term (NU)
};
static_assert(BaSize<6>::JD == 20 && BaSize<6>::PV == 54, "the header states the NC = 6 scratch");
static_assert(BaSize<9>::JD == 26 && BaSize<9>::PV == 108, "the header states the NC = 9 scratch");

// A used observation: its track, image, member and pixel position.
struct BaObs {
  int k, a, m, pad;
  float x, y;
};

// The intrinsic state of a camera that refines them (NC = 9); nothing for NC = 6.
template <int NC>
struct BaIntr {};
template <>
struct BaIntr<9> {
  double Kc[6];                      // candidate K[0..5]
  double k[2], kc[2];                // (k1, k2): current, candidate
  int refine, pad;                   // bits 0 focal, 1 k1, 2 k2
};

// A camera: the input, the state of the LM loop and its sorted observations [start, end).
template <int NC>
struct BaCam : BaIntr<NC> {
  double K[6];                       // K[0..5] of the row-major K (K[3] unused); current
  double R[9], t[3];                 // current
  double Rc[9], tc[3];               // candidate
  double P[12];                      // K [R | t] of the final parameters (outputs)
  double U[BaSize<NC>::NU];          // U* (damped), upper triangle row by row; held rows and columns are identity
  double L[BaSize<NC>::NU];          // Cholesky factor of the preconditioner block, lower triangle row by row
  double x[NC], r[NC], z[NC], p[NC], q[NC];
  const SiftPoint *pts;
  int n, fixed, mask, start, end, pad;
};

static_assert(sizeof(BaCam<6>) == 944, "the header states the per-image scratch");
static_assert(sizeof(BaCam<9>) == 1536, "the header states the per-image scratch");

// A track's point: current, candidate, and the damped V* factor, gradient and CG scratch.
struct BaPt {
  double X[3], Xc[3];
  double L[6];                       // Cholesky factor of V*, lower triangle row by row
  double g[3], q[3], y[3];           // J_p^T r, V*^-1 g, V*^-1 W^T p
};

// The words the host reads back.
struct BaResult {
  double cost[2];
  unsigned long long stats[8];
  unsigned long long accepted;
};

template <int NC>
struct BaParams {
  BaCam<NC> *cams;
  BaPt *pts;
  const int *offsets;
  const int2 *members;
  const unsigned char *use;
  double *points;
  float *errors;
  unsigned char *inlier;
  int *cnt;                          // [numTracks + 1]: used observations of a participating track, else 0
  int *start;                        // [numTracks + 1]: exclusive sum of cnt
  BaObs *obs;                        // [numMembers]
  double *J;                         // [numMembers][JD]
  int *keys, *vals;                  // [numMembers]: image and observation, sorted in keysS / order
  const int *keysS, *order;
  double *pieces;                    // [tiles + numImages][PV]
  double *camPart;                   // [ceil(numImages / 32)][BA_CP]: r.r (or b~.b~), r.z, p.S p
  double *ptPart;                    // [ceil(numTracks / 256)][2]
  unsigned int *flags;               // [maxIterations]: bit 0 a Cholesky pivot failed, bit 1 a refined focal <= 0
  double *trace;                     // [maxIterations][4]
  BaResult *res;
  double thr2, tol2;
  int numImages, numTracks, numMembers, maxIterations, maxLinear;
  int loss;                          // robust kernels: 1 soft-L1, 2 Cauchy
  double c2;                         // robust kernels: the squared loss scale
};

// ---- small dense helpers (row-major full matrices in registers) ----------------------------------------------------

// The free components of a camera with fixed code f: 0 all six, 1 none, 2..4 all but t[f - 2] (bits 0-2 w, 3-5 t).
__device__ __forceinline__ int ba_free_mask(int f) { return f == 0 ? 0x3f : f == 1 ? 0 : 0x3f & ~(1 << (f + 1)); }

__device__ __forceinline__ double ba_depth(const double *R, const double *t, const double (&X)[3])
{
  return R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + t[2];
}

// The residual of an observation at (R, t, X) into r; J (when given) receives J_c's two rows (w then delta), J_p's two
// rows and r.  Returns the depth.
__device__ __forceinline__ double ba_linearise(const double *K, const double *R, const double *t, const double (&X)[3],
                                               float x, float y, double (&r)[2], double *J)
{
  double RX[3];
#pragma unroll
  for (int i = 0; i < 3; i++) RX[i] = R[3 * i] * X[0] + R[3 * i + 1] * X[1] + R[3 * i + 2] * X[2];
  const double z = RX[2] + t[2], a = (RX[0] + t[0]) / z, b = (RX[1] + t[1]) / z;
  r[0] = K[0] * a + K[1] * b + K[2] - (double)x;
  r[1] = K[4] * b + K[5] - (double)y;
  if (J) {
    const double gr[2][3] = {{K[0] / z, K[1] / z, -(K[0] * a + K[1] * b) / z}, {0.0, K[4] / z, -K[4] * b / z}};
#pragma unroll
    for (int q = 0; q < 2; q++) {
      const double *g = gr[q];
      J[6 * q + 0] = RX[1] * g[2] - RX[2] * g[1];
      J[6 * q + 1] = RX[2] * g[0] - RX[0] * g[2];
      J[6 * q + 2] = RX[0] * g[1] - RX[1] * g[0];
#pragma unroll
      for (int i = 0; i < 3; i++) J[6 * q + 3 + i] = g[i];
#pragma unroll
      for (int j = 0; j < 3; j++) J[12 + 3 * q + j] = g[0] * R[j] + g[1] * R[3 + j] + g[2] * R[6 + j];
    }
    J[18] = r[0];
    J[19] = r[1];
  }
  return z;
}

// The same under radial distortion k = (k1, k2) (the header's camera model): J (when given) receives J_c's two rows
// (w, delta, f, k1, k2), J_p's two rows and r.  The pose and point rows go through the distortion's 2 x 2 derivative.
__device__ __forceinline__ double ba_linearise_radial(const double *K, const double *k, const double *R,
                                                      const double *t, const double (&X)[3], float x, float y,
                                                      double (&r)[2], double *J)
{
  double RX[3];
#pragma unroll
  for (int i = 0; i < 3; i++) RX[i] = R[3 * i] * X[0] + R[3 * i + 1] * X[1] + R[3 * i + 2] * X[2];
  const double z = RX[2] + t[2], a = (RX[0] + t[0]) / z, b = (RX[1] + t[1]) / z;
  const double rho2 = a * a + b * b, D = 1.0 + rho2 * (k[0] + k[1] * rho2);
  const double ad = D * a, bd = D * b;
  const double pu = K[0] * ad + K[1] * bd, pv = K[4] * bd;
  r[0] = pu + K[2] - (double)x;
  r[1] = pv + K[5] - (double)y;
  if (J) {
    const double Dp = 2.0 * (k[0] + 2.0 * k[1] * rho2);      // 2 dD / d(rho^2)
    const double Daa = D + Dp * a * a, Dab = Dp * a * b, Dbb = D + Dp * b * b;
    // d(u, v) / d(a, b) = [K0 K1; 0 K4] d(a', b') / d(a, b), then gr = d(u, v) / d(a, b) d(a, b) / d(Xc)
    const double du[2][2] = {{K[0] * Daa + K[1] * Dab, K[0] * Dab + K[1] * Dbb}, {K[4] * Dab, K[4] * Dbb}};
#pragma unroll
    for (int q = 0; q < 2; q++) {
      const double g[3] = {du[q][0] / z, du[q][1] / z, -(du[q][0] * a + du[q][1] * b) / z};
      J[9 * q + 0] = RX[1] * g[2] - RX[2] * g[1];
      J[9 * q + 1] = RX[2] * g[0] - RX[0] * g[2];
      J[9 * q + 2] = RX[0] * g[1] - RX[1] * g[0];
#pragma unroll
      for (int i = 0; i < 3; i++) J[9 * q + 3 + i] = g[i];
#pragma unroll
      for (int j = 0; j < 3; j++) J[18 + 3 * q + j] = g[0] * R[j] + g[1] * R[3 + j] + g[2] * R[6 + j];
    }
    const double eu = K[0] * a + K[1] * b, ev = K[4] * b;    // d(u, v) / d(k1) = (eu, ev) rho^2
    J[6] = pu / K[0];
    J[15] = pv / K[0];
    J[7] = eu * rho2;
    J[16] = ev * rho2;
    J[8] = J[7] * rho2;
    J[17] = J[16] * rho2;
    J[24] = r[0];
    J[25] = r[1];
  }
  return z;
}

// The observation's residual at a camera's current or candidate parameters (J as ba_linearise).
template <int NC>
__device__ __forceinline__ double ba_observe(const BaCam<NC> &c, bool cand, const double (&X)[3], float x, float y,
                                             double (&r)[2], double *J)
{
  if constexpr (NC == 6)
    return ba_linearise(c.K, cand ? c.Rc : c.R, cand ? c.tc : c.t, X, x, y, r, J);
  else
    return ba_linearise_radial(cand ? c.Kc : c.K, cand ? c.kc : c.k, cand ? c.Rc : c.R, cand ? c.tc : c.t, X, x, y,
                               r, J);
}

// ---- setup kernels --------------------------------------------------------------------------------------------------

// The used observations of track k (through f(m, a, x, y)); -1 for a malformed track.
template <int NC, class F>
__device__ __forceinline__ int ba_used(const BaParams<NC> &p, int k, int &invalid, F &&f)
{
  const int lo = p.offsets[k], hi = p.offsets[k + 1];
  if (lo < 0 || hi < lo || hi > p.numMembers) return -1;
  const double X[3] = {p.points[3 * (size_t)k], p.points[3 * (size_t)k + 1], p.points[3 * (size_t)k + 2]};
  const bool finite = isfinite(X[0]) && isfinite(X[1]) && isfinite(X[2]);
  int used = 0;
  invalid = 0;
  for (int m = lo; m < hi; m++) {
    float x, y;
    const int2 af = p.members[m];
    if (!tr_member(p.cams, p.numImages, af, x, y)) { invalid++; continue; }
    if (!finite || (p.use && !p.use[m])) continue;
    const BaCam<NC> &c = p.cams[af.x];
    if (!(ba_depth(c.R, c.t, X) > 0.0)) continue;
    f(m, af.x, x, y, used);
    used++;
  }
  return used;
}

template <int NC>
__global__ void __launch_bounds__(BA_THREADS) bundle_count_kernel(BaParams<NC> p)
{
  co_count(p, blockIdx.x * BA_THREADS + threadIdx.x, [&](int k, int &invalid) {
    return ba_used(p, k, invalid, [](int, int, float, float, int) {});
  });
}

template <int NC>
__global__ void __launch_bounds__(BA_THREADS) bundle_fill_kernel(BaParams<NC> p)
{
  const int i = blockIdx.x * BA_THREADS + threadIdx.x;
  const int N = p.start[p.numTracks];
  if (i >= N && i < p.numMembers) {                          // past the observations: sorted last
    p.keys[i] = p.numImages;
    p.vals[i] = i;
  }
  if (i >= p.numTracks || p.cnt[i] == 0) return;
  const int k = i, s = p.start[k];
  int invalid = 0;
  ba_used(p, k, invalid, [&](int m, int a, float x, float y, int j) {
    p.obs[s + j] = BaObs{k, a, m, 0, x, y};
    p.keys[s + j] = a;
    p.vals[s + j] = s + j;
  });
#pragma unroll
  for (int j = 0; j < 3; j++) p.pts[k].X[j] = p.points[3 * (size_t)k + j];
}

// ---- the cooperative kernel ---------------------------------------------------------------------------------------

// J_c^T (J_p y) of observation o (NC values)
template <int NC>
__device__ __forceinline__ void ba_wy(const double *J, const double *y, double *v)
{
  constexpr int P = 2 * NC;
  const double s0 = J[P] * y[0] + J[P + 1] * y[1] + J[P + 2] * y[2];
  const double s1 = J[P + 3] * y[0] + J[P + 4] * y[1] + J[P + 5] * y[2];
#pragma unroll
  for (int i = 0; i < NC; i++) v[i] = J[i] * s0 + J[NC + i] * s1;
}

// J_p^T (J_c x), accumulated into h (3 values)
template <int NC>
__device__ __forceinline__ void ba_wtx(const double *J, const double *x, double (&h)[3])
{
  constexpr int P = 2 * NC;
  double s0 = 0.0, s1 = 0.0;
#pragma unroll
  for (int i = 0; i < NC; i++) { s0 += J[i] * x[i]; s1 += J[NC + i] * x[i]; }
#pragma unroll
  for (int j = 0; j < 3; j++) h[j] += J[P + j] * s0 + J[P + 3 + j] * s1;
}

// the packed upper-triangle index of (i, j), i <= j, of an N x N matrix
template <int N>
__device__ __forceinline__ int ba_up(int i, int j) { return i * N - i * (i - 1) / 2 + (j - i); }

// Linearise every observation of track k at the current parameters (or the candidate ones); returns its cost.  Under a
// robust loss the observation's r and Jacobian rows are scaled by sqrt(rho'), the cost is c^2 rho(s / c^2).
template <int NC, bool ROBUST>
__device__ __forceinline__ double ba_relinearise(const BaParams<NC> &p, int k, int s, int e, bool cand)
{
  constexpr int JD = BaSize<NC>::JD;
  const BaPt &pt = p.pts[k];
  const double X[3] = {cand ? pt.Xc[0] : pt.X[0], cand ? pt.Xc[1] : pt.X[1], cand ? pt.Xc[2] : pt.X[2]};
  double cost = 0.0;
  for (int o = s; o < e; o++) {
    const BaObs ob = p.obs[o];
    const BaCam<NC> &c = p.cams[ob.a];
    double r[2];
    double *J = p.J + (size_t)o * JD;
    ba_observe<NC>(c, cand, X, ob.x, ob.y, r, J);
    if constexpr (ROBUST) {
      double w2;
      cost += vp_loss(p.loss, p.c2, r[0] * r[0] + r[1] * r[1], &w2);
      const double w = sqrt(w2);
#pragma unroll
      for (int j = 0; j < JD; j++) J[j] *= w;
    } else {
      cost += r[0] * r[0] + r[1] * r[1];
    }
  }
  return cost;
}

template <int NC, bool ROBUST>
__global__ void __launch_bounds__(BA_THREADS) bundle_kernel(BaParams<NC> p)
{
  constexpr int NU = BaSize<NC>::NU, JD = BaSize<NC>::JD, PV = BaSize<NC>::PV, PJ = 2 * NC;   // PJ: J_p's first entry
  cg::grid_group grid = cg::this_grid();
  const int tid = (int)(blockIdx.x * BA_THREADS + threadIdx.x), nthreads = (int)gridDim.x * BA_THREADS;
  const int lane = (int)threadIdx.x & 31;
  const int warpG = tid >> 5, numWarps = nthreads >> 5;
  const int C = p.numImages, N = p.start[p.numTracks];
  const int camTiles = (C + 31) / 32, ptTiles = (p.numTracks + BA_THREADS - 1) / BA_THREADS;

  // 0. every camera's sorted range, its free components; the linearisation at the input and its cost
  co_ranges(p.keysS, N, p.cams, tid, nthreads);
  grid.sync();
  for (int a = tid; a < C; a += nthreads) {
    BaCam<NC> &c = p.cams[a];
    if constexpr (NC == 6)
      c.mask = c.end > c.start ? ba_free_mask(c.fixed) : 0;
    else
      c.mask = c.end > c.start ? ba_free_mask(c.fixed) | (c.refine << 6) : 0;
    if (c.mask) atomicAdd(&p.res->stats[5], (unsigned long long)__popc(c.mask));
  }
  co_per_track<1, BA_THREADS>(p.start, p.numTracks, p.ptPart, [&](int k, int s, int e, double *v) {
    v[0] = ba_relinearise<NC, ROBUST>(p, k, s, e, false);
  });
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
    // A. per point: V* (damped) by Cholesky, g_p = J_p^T r, q = V*^-1 g_p
    co_per_track<0, BA_THREADS>(p.start, p.numTracks, nullptr, [&](int k, int s, int e, double *) {
      double V[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, g[3] = {0, 0, 0};
      for (int o = s; o < e; o++) {
        const double *J = p.J + (size_t)o * JD;
#pragma unroll
        for (int q = 0; q < 2; q++) {
          const double *jp = J + PJ + 3 * q, r = J[PJ + 6 + q];
#pragma unroll
          for (int i = 0; i < 3; i++) {
#pragma unroll
            for (int j = i; j < 3; j++) V[i][j] += jp[i] * jp[j];
            g[i] += jp[i] * r;
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 3; i++) {
        V[i][i] += vp_damping(V[i][i], lam);
#pragma unroll
        for (int j = 0; j < i; j++) V[i][j] = V[j][i];
      }
      BaPt &pt = p.pts[k];
      if (!vp_chol<3>(V, pt.L)) { atomicOr(&p.flags[it], 1u); return; }
      double q[3];
      vp_chol_solve<3>(pt.L, g, q);
#pragma unroll
      for (int i = 0; i < 3; i++) { pt.g[i] = g[i]; pt.q[i] = q[i]; }
    });
    grid.sync();
    unsigned int fail = *(volatile unsigned int *)&p.flags[it];

    // B. the camera pieces: U, g_c, W q and the Schur term W_o V*^-1 W_ak^T (W_ak: the track's observations in image a)
    if (!fail) {
      co_pieces<NU, 0, PV, BA_THREADS>(p.keysS, p.order, p.pieces, N, p.cams, [&](int o, int, double *v) {
        const double *J = p.J + (size_t)o * JD;
        int n = 0;
#pragma unroll
        for (int i = 0; i < NC; i++)
#pragma unroll
          for (int j = i; j < NC; j++) v[n++] = J[i] * J[j] + J[NC + i] * J[NC + j];
      });
      co_pieces<2 * NC, NU, PV, BA_THREADS>(p.keysS, p.order, p.pieces, N, p.cams, [&](int o, int, double *v) {
        const double *J = p.J + (size_t)o * JD;
        const double *q = p.pts[p.obs[o].k].q;
#pragma unroll
        for (int i = 0; i < NC; i++) v[i] = J[i] * J[PJ + 6] + J[NC + i] * J[PJ + 7];
        ba_wy<NC>(J, q, v + NC);
      });
      co_pieces<NU, NU + 2 * NC, PV, BA_THREADS>(p.keysS, p.order, p.pieces, N, p.cams, [&](int o, int a, double *v) {
        const double *J = p.J + (size_t)o * JD;
        const int k = p.obs[o].k;
        double Wo[NC][3], Wa[NC][3], Y[NC][3];
#pragma unroll
        for (int i = 0; i < NC; i++)
#pragma unroll
          for (int j = 0; j < 3; j++) {
            Wo[i][j] = J[i] * J[PJ + j] + J[NC + i] * J[PJ + 3 + j];
            Wa[i][j] = 0.0;
          }
        for (int u = p.start[k]; u < p.start[k + 1]; u++) {
          if (p.obs[u].a != a) continue;
          const double *Ju = p.J + (size_t)u * JD;
#pragma unroll
          for (int i = 0; i < NC; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) Wa[i][j] += Ju[i] * Ju[PJ + j] + Ju[NC + i] * Ju[PJ + 3 + j];
        }
        const double *L = p.pts[k].L;
#pragma unroll
        for (int i = 0; i < NC; i++) vp_chol_solve<3>(L, Wa[i], Y[i]);
        int n = 0;
#pragma unroll
        for (int i = 0; i < NC; i++)
#pragma unroll
          for (int j = i; j < NC; j++) v[n++] = Wo[i][0] * Y[j][0] + Wo[i][1] * Y[j][1] + Wo[i][2] * Y[j][2];
      });
    }
    grid.sync();

    // C. per camera (a lane each): U*, the right-hand side b~ = -g_c + W q, the preconditioner block and its factor;
    // x = 0, r = b~, z = M^-1 r, p = 0; the partials of b~.b~ and r.z
    if (!fail)
      for (int w = warpG; w < camTiles; w += numWarps) {
        const int a = w * 32 + lane;
        double d[2] = {0.0, 0.0};
        if (a < C) {
          BaCam<NC> &c = p.cams[a];
          double U[NU], G[2 * NC], T[NU];
          co_gather<NU, 0, PV>(p.pieces, a, c, U);
          co_gather<2 * NC, NU, PV>(p.pieces, a, c, G);
          co_gather<NU, NU + 2 * NC, PV>(p.pieces, a, c, T);
          double Us[NC][NC], M[NC][NC];
#pragma unroll
          for (int i = 0; i < NC; i++)
#pragma unroll
            for (int j = i; j < NC; j++) {
              const bool fr = ((c.mask >> i) & 1) && ((c.mask >> j) & 1);
              double u = U[ba_up<NC>(i, j)];
              if (i == j) u += vp_damping(u, lam);
              Us[i][j] = Us[j][i] = fr ? u : (i == j ? 1.0 : 0.0);
              M[i][j] = M[j][i] = fr ? u - T[ba_up<NC>(i, j)] : (i == j ? 1.0 : 0.0);
            }
#pragma unroll
          for (int i = 0; i < NC; i++)
#pragma unroll
            for (int j = i; j < NC; j++) c.U[ba_up<NC>(i, j)] = Us[i][j];
          if (!vp_chol<NC>(M, c.L)) {
            atomicOr(&p.flags[it], 1u);
          } else {
            double r[NC], z[NC];
#pragma unroll
            for (int i = 0; i < NC; i++) r[i] = ((c.mask >> i) & 1) ? -G[i] + G[NC + i] : 0.0;
            vp_chol_solve<NC>(c.L, r, z);
#pragma unroll
            for (int i = 0; i < NC; i++) {
              c.x[i] = 0.0; c.r[i] = r[i]; c.z[i] = z[i]; c.p[i] = 0.0;
              d[0] += r[i] * r[i];
              d[1] += r[i] * z[i];
            }
          }
        }
        co_warp_partial<2>(d, p.camPart + BA_CP * (size_t)w);
      }
    grid.sync();
    fail = *(volatile unsigned int *)&p.flags[it];

    // D-G. preconditioned CG on S dc = b~ from dc = 0
    int cgIt = 0;
    if (!fail) {
      double t2[2];
      co_totals<2>(p.camPart, camTiles, BA_CP, t2);
      const double thr = p.tol2 * t2[0];
      double rr = t2[0], rz = t2[1], beta = 0.0;
      while (cgIt < p.maxLinear && !(rr <= thr)) {
        // D. per point: y = V*^-1 W^T p, with p = z + beta p_old of each camera
        co_per_track<0, BA_THREADS>(p.start, p.numTracks, nullptr, [&](int k, int s, int e, double *) {
          double h[3] = {0.0, 0.0, 0.0};
          for (int o = s; o < e; o++) {
            const BaCam<NC> &c = p.cams[p.obs[o].a];
            double pe[NC];
#pragma unroll
            for (int i = 0; i < NC; i++) pe[i] = fma(beta, c.p[i], c.z[i]);
            ba_wtx<NC>(p.J + (size_t)o * JD, pe, h);
          }
          BaPt &pt = p.pts[k];
          double y[3];
          vp_chol_solve<3>(pt.L, h, y);
#pragma unroll
          for (int i = 0; i < 3; i++) pt.y[i] = y[i];
        });
        grid.sync();
        // E. the camera pieces of W y
        co_pieces<NC, 0, PV, BA_THREADS>(p.keysS, p.order, p.pieces, N, p.cams, [&](int o, int, double *v) {
          ba_wy<NC>(p.J + (size_t)o * JD, p.pts[p.obs[o].k].y, v);
        });
        grid.sync();
        // F. per camera: p = z + beta p_old, q = S p = U* p - W y (held components 0); the partials of p.q
        for (int w = warpG; w < camTiles; w += numWarps) {
          const int a = w * 32 + lane;
          double d[1] = {0.0};
          if (a < C) {
            BaCam<NC> &c = p.cams[a];
            double Wy[NC], pn[NC];
            co_gather<NC, 0, PV>(p.pieces, a, c, Wy);
#pragma unroll
            for (int i = 0; i < NC; i++) pn[i] = fma(beta, c.p[i], c.z[i]);
#pragma unroll
            for (int i = 0; i < NC; i++) {
              double s = 0.0;
#pragma unroll
              for (int j = 0; j < NC; j++) s += c.U[ba_up<NC>(min(i, j), max(i, j))] * pn[j];
              const double q = ((c.mask >> i) & 1) ? s - Wy[i] : 0.0;
              c.p[i] = pn[i];
              c.q[i] = q;
              d[0] += pn[i] * q;
            }
          }
          co_warp_partial<1>(d, p.camPart + BA_CP * (size_t)w + 2);
        }
        grid.sync();
        double pq[1];
        co_totals<1>(p.camPart + 2, camTiles, BA_CP, pq);
        if (!(pq[0] > 0.0)) break;
        const double alpha = rz / pq[0];
        // G. per camera: x += alpha p, r -= alpha q, z = M^-1 r; the partials of r.r and r.z
        for (int w = warpG; w < camTiles; w += numWarps) {
          const int a = w * 32 + lane;
          double d[2] = {0.0, 0.0};
          if (a < C) {
            BaCam<NC> &c = p.cams[a];
            double r[NC], z[NC];
#pragma unroll
            for (int i = 0; i < NC; i++) {
              c.x[i] = fma(alpha, c.p[i], c.x[i]);
              r[i] = fma(-alpha, c.q[i], c.r[i]);
              c.r[i] = r[i];
            }
            vp_chol_solve<NC>(c.L, r, z);
#pragma unroll
            for (int i = 0; i < NC; i++) {
              c.z[i] = z[i];
              d[0] += r[i] * r[i];
              d[1] += r[i] * z[i];
            }
          }
          co_warp_partial<2>(d, p.camPart + BA_CP * (size_t)w);
        }
        cgIt++;
        grid.sync();
        co_totals<2>(p.camPart, camTiles, BA_CP, t2);
        rr = t2[0];
        beta = t2[1] / rz;
        rz = t2[1];
      }
    }
    cgTotal += cgIt;

    // H. back-substitution dp = V*^-1 (-g_p - W^T dc) and the candidate points; the candidate cameras
    double cand[2] = {CUDART_NAN, 0.0};
    bool badFocal = false;
    if (!fail) {
      co_per_track<0, BA_THREADS>(p.start, p.numTracks, nullptr, [&](int k, int s, int e, double *) {
        BaPt &pt = p.pts[k];
        double h[3] = {0.0, 0.0, 0.0}, dp[3];
        for (int o = s; o < e; o++) ba_wtx<NC>(p.J + (size_t)o * JD, p.cams[p.obs[o].a].x, h);
#pragma unroll
        for (int i = 0; i < 3; i++) h[i] = -pt.g[i] - h[i];
        vp_chol_solve<3>(pt.L, h, dp);
#pragma unroll
        for (int i = 0; i < 3; i++) pt.Xc[i] = pt.X[i] + dp[i];
      });
      for (int a = tid; a < C; a += nthreads) {
        BaCam<NC> &c = p.cams[a];
        if constexpr (NC == 9) {
          // f <- f + df with K1 / K0 and K4 / K0 held; k <- k + dk
#pragma unroll
          for (int i = 0; i < 6; i++) c.Kc[i] = c.K[i];
          if ((c.mask >> 6) & 1) {
            const double f = c.K[0] + c.x[6], s = f / c.K[0];
            c.Kc[0] = f;
            c.Kc[1] = c.K[1] * s;
            c.Kc[4] = c.K[4] * s;
            if (!(f > 0.0)) atomicOr(&p.flags[it], 2u);
          }
#pragma unroll
          for (int i = 0; i < 2; i++) c.kc[i] = ((c.mask >> (7 + i)) & 1) ? c.k[i] + c.x[7 + i] : c.k[i];
        }
        if (!(NC == 6 ? c.mask : c.mask & 0x3f)) {               // no free pose component
#pragma unroll
          for (int i = 0; i < 9; i++) c.Rc[i] = c.R[i];
#pragma unroll
          for (int i = 0; i < 3; i++) c.tc[i] = c.t[i];
          continue;
        }
        double Q[9];
        vp_rotate(c.x, c.R, c.Rc, Q);
#pragma unroll
        for (int i = 0; i < 3; i++) c.tc[i] = ((c.mask >> (3 + i)) & 1) ? c.t[i] + c.x[3 + i] : c.t[i];
      }
      grid.sync();
      if constexpr (NC == 9) badFocal = (*(volatile unsigned int *)&p.flags[it] & 2u) != 0;
      // I. the candidate's cost and its observations behind a camera
      co_per_track<2, BA_THREADS>(p.start, p.numTracks, p.ptPart, [&](int k, int s, int e, double *v) {
        const BaPt &pt = p.pts[k];
        const double X[3] = {pt.Xc[0], pt.Xc[1], pt.Xc[2]};
        for (int o = s; o < e; o++) {
          const BaObs ob = p.obs[o];
          const BaCam<NC> &c = p.cams[ob.a];
          double r[2];
          const double z = ba_observe<NC>(c, true, X, ob.x, ob.y, r, nullptr);
          if constexpr (ROBUST)
            v[0] += vp_loss(p.loss, p.c2, r[0] * r[0] + r[1] * r[1], nullptr);
          else
            v[0] += r[0] * r[0] + r[1] * r[1];
          if (!(z > 0.0)) v[1] += 1.0;
        }
      });
      grid.sync();
      co_totals<2>(p.ptPart, ptTiles, 2, cand);
    }

    // J. accept or reject
    const bool accept = !fail && !badFocal && cand[1] == 0.0 && cand[0] < cost;
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
      for (int a = tid; a < C; a += nthreads) {
        BaCam<NC> &c = p.cams[a];
#pragma unroll
        for (int i = 0; i < 9; i++) c.R[i] = c.Rc[i];
#pragma unroll
        for (int i = 0; i < 3; i++) c.t[i] = c.tc[i];
        if constexpr (NC == 9) {
#pragma unroll
          for (int i = 0; i < 6; i++) c.K[i] = c.Kc[i];
          c.k[0] = c.kc[0];
          c.k[1] = c.kc[1];
        }
      }
      co_per_track<0, BA_THREADS>(p.start, p.numTracks, nullptr, [&](int k, int s, int e, double *) {
        ba_relinearise<NC, ROBUST>(p, k, s, e, true);
        BaPt &pt = p.pts[k];
#pragma unroll
        for (int i = 0; i < 3; i++) pt.X[i] = pt.Xc[i];
      });
      grid.sync();
      if (stop) break;
    } else {
      lam *= 10.0;
      if (lam > 1e16) break;
    }
  }

  // K. the outputs: P = K [R | t] of every camera; the points; per member the error and inlier byte
  for (int a = tid; a < C; a += nthreads) {
    BaCam<NC> &c = p.cams[a];
    const double K9[9] = {c.K[0], c.K[1], c.K[2], 0.0, c.K[4], c.K[5], 0.0, 0.0, 1.0};
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const double col[3] = {j < 3 ? c.R[j] : c.t[0], j < 3 ? c.R[3 + j] : c.t[1], j < 3 ? c.R[6 + j] : c.t[2]};
        c.P[4 * i + j] = K9[3 * i] * col[0] + K9[3 * i + 1] * col[1] + K9[3 * i + 2] * col[2];
      }
  }
  grid.sync();
  for (int k = tid; k < p.numTracks; k += nthreads) {
    const int lo = p.offsets[k], hi = p.offsets[k + 1];
    if (lo < 0 || hi < lo || hi > p.numMembers) continue;
    double X[3];
    const bool moved = p.start[k + 1] > p.start[k];
#pragma unroll
    for (int i = 0; i < 3; i++) {
      X[i] = moved ? p.pts[k].X[i] : p.points[3 * (size_t)k + i];
      if (moved) p.points[3 * (size_t)k + i] = X[i];
    }
    if (!p.errors && !p.inlier) continue;
    const bool has = isfinite(X[0]) && isfinite(X[1]) && isfinite(X[2]);
    for (int m = lo; m < hi; m++) {
      float x, y, err = CUDART_NAN_F;
      unsigned char in = 0;
      const int2 af = p.members[m];
      if (tr_member(p.cams, C, af, x, y) && has) {
        if constexpr (NC == 6) {
          tr_reproject(p.cams[af.x].P, X, x, y, p.thr2, err, in);
        } else {
          // the pixel error under the final intrinsics, distortion included (inf behind the camera)
          double r[2];
          const double z = ba_observe<NC>(p.cams[af.x], false, X, x, y, r, nullptr);
          const double e2 = r[0] * r[0] + r[1] * r[1];
          in = z > 0.0 && e2 < p.thr2;
          err = z > 0.0 ? (float)sqrt(e2) : CUDART_INF_F;
        }
      }
      if (p.errors) p.errors[m] = err;
      if (p.inlier) p.inlier[m] = in;
    }
  }
  if (tid == 0) {
    p.res->cost[0] = cost0;
    p.res->cost[1] = cost;
    p.res->accepted = accepted;
    p.res->stats[6] = lmIters;
    p.res->stats[7] = cgTotal;
  }
}

// ---- undistortion of records ----------------------------------------------------------------------------------------

// An image of cs_undistort_records: its K[0..5], (k1, k2), its records in and out, and its first record's global index.
struct UdImage {
  double K[6], k[2];
  const SiftPoint *in;
  SiftPoint *out;
  long long first;
  int n, pad;
};

constexpr int UD_THREADS = 256;
constexpr int UD_NEWTON = 20;        // Newton iterations at most

// The undistorted position of (x, y) under K and k (the header's rule at cs_undistort_records); NaN when the solve
// does not converge or the derivative is not > 0 at its root.
__device__ __forceinline__ void ud_point(const double *K, const double *k, float x, float y, float &xo, float &yo)
{
  const double b = ((double)y - K[5]) / K[4], a = ((double)x - K[2] - K[1] * b) / K[0];
  const double rd = sqrt(a * a + b * b);
  double ru = rd, s = 1.0;
  bool ok = false;
  for (int it = 0; it < UD_NEWTON; it++) {
    const double r2 = ru * ru, d = 1.0 + r2 * (3.0 * k[0] + 5.0 * k[1] * r2);
    if (!(d > 0.0)) break;
    const double step = (ru * (1.0 + r2 * (k[0] + k[1] * r2)) - rd) / d;
    ru -= step;
    if (fabs(step) <= 1e-12 * rd) { ok = true; break; }
  }
  const double r2 = ru * ru;
  ok = ok && 1.0 + r2 * (3.0 * k[0] + 5.0 * k[1] * r2) > 0.0;
  if (rd > 0.0) s = ru / rd;
  const double au = a * s, bu = b * s;
  xo = ok ? (float)(K[0] * au + K[1] * bu + K[2]) : CUDART_NAN_F;
  yo = ok ? (float)(K[4] * bu + K[5]) : CUDART_NAN_F;
}

// One thread per record of every image: the image by binary search over the first indices, the record copied word by
// word (unless in place), then its corrected position.
__global__ void __launch_bounds__(UD_THREADS) undistort_kernel(const UdImage *imgs, int numImages, long long total)
{
  const long long g = (long long)blockIdx.x * UD_THREADS + threadIdx.x;
  if (g >= total) return;
  int lo = 0, hi = numImages - 1;
  while (lo < hi) {                                          // the last image with first <= g
    const int mid = (lo + hi + 1) >> 1;
    if (imgs[mid].first <= g) lo = mid; else hi = mid - 1;
  }
  const UdImage &im = imgs[lo];
  const int f = (int)(g - im.first);
  const SiftPoint *src = im.in + f;
  SiftPoint *dst = im.out + f;
  const float x = src->xpos, y = src->ypos;
  if (dst != src) {
    const unsigned int *s = reinterpret_cast<const unsigned int *>(src);
    unsigned int *d = reinterpret_cast<unsigned int *>(dst);
    for (int w = 0; w < (int)(sizeof(SiftPoint) / 4); w++) d[w] = s[w];
  }
  float xo, yo;
  ud_point(im.K, im.k, x, y, xo, yo);
  dst->xpos = xo;
  dst->ypos = yo;
}

// The pinned layout: the result words, the trace, then the camera table of NC; returns the table's offset.
template <int NC>
size_t bundle_host_layout(int numImages, int maxIterations, size_t *bytes)
{
  Layout H(256);
  H.take(sizeof(BaResult));
  H.take((size_t)maxIterations * 4 * sizeof(double));
  const size_t camAt = H.take((size_t)numImages * sizeof(BaCam<NC>));
  if (bytes) *bytes = H.bytes;
  return camAt;
}

template <int NC, bool ROBUST>
int bundle_run(DeviceCtx &c, const cs_match_set *sets, int numImages, const double *Ks, const double *dists,
               const unsigned char *refine, int loss, double lossScale, const double *Rs, const double *ts,
               const unsigned char *fixed, const int *offsets, int numTracks, const int *members, int numMembers,
               const unsigned char *use, double *points, int maxIterations, int maxLinearIterations, double linearTol,
               double maxError, float *errors, unsigned char *inlier)
{
  constexpr int JD = BaSize<NC>::JD, PV = BaSize<NC>::PV;
  const int M = numMembers, T = numTracks, C = numImages;
  const int tiles = idivup(M, CO_TILE);
  const int bits = radix_bits(C);                                  // every key, the sentinel C included
  size_t scanBytes = 0, sortBytes = 0;
  CS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scanBytes, (int *)nullptr, (int *)nullptr, T + 1, c.stream));
  CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sortBytes, (int *)nullptr, (int *)nullptr, (int *)nullptr,
                                          (int *)nullptr, std::max(M, 1), 0, bits, c.stream));

  // device scratch (header: cs_bundle_adjust)
  Layout L(256);
  const size_t resAt = L.take(sizeof(BaResult)), traceAt = L.take((size_t)maxIterations * 4 * sizeof(double));
  const size_t flagsAt = L.take((size_t)maxIterations * sizeof(unsigned int)), zeroEnd = L.bytes;
  const size_t camAt = L.take((size_t)C * sizeof(BaCam<NC>)), ptAt = L.take((size_t)T * sizeof(BaPt));
  const size_t cntAt = L.take(((size_t)T + 1) * sizeof(int)), startAt = L.take(((size_t)T + 1) * sizeof(int));
  const size_t obsAt = L.take((size_t)M * sizeof(BaObs)), jAt = L.take((size_t)M * JD * sizeof(double));
  const size_t keysAt = L.take((size_t)M * sizeof(int)), valsAt = L.take((size_t)M * sizeof(int));
  const size_t keysSAt = L.take((size_t)M * sizeof(int)), orderAt = L.take((size_t)M * sizeof(int));
  const size_t piecesAt = L.take(((size_t)tiles + C) * PV * sizeof(double));
  const size_t camPartAt = L.take((size_t)idivup(C, 32) * BA_CP * sizeof(double));
  const size_t ptPartAt = L.take((size_t)idivup(T, BA_THREADS) * 2 * sizeof(double));
  const size_t tempAt = L.take(std::max(scanBytes, sortBytes));
  int r = c.bundle.grow(L.bytes);
  if (r < 0) return r;
  char *base = c.bundle.as<char>();

  // pinned: the result words and the trace (copied back), then the camera table (uploaded, then copied back)
  // (the same offsets as the device's result words and trace, so that one copy brings both back)
  size_t hBytes = 0;
  const size_t hCamAt = bundle_host_layout<NC>(C, maxIterations, &hBytes);
  if ((r = c.h_bundle.grow(hBytes)) < 0) return r;
  BaCam<NC> *cams = reinterpret_cast<BaCam<NC> *>(c.h_bundle.as<char>() + hCamAt);
  for (int a = 0; a < C; a++) {
    BaCam<NC> &m = cams[a];
    memset(&m, 0, sizeof m);
    for (int i = 0; i < 6; i++) m.K[i] = Ks[9 * (size_t)a + i];
    for (int i = 0; i < 9; i++) m.R[i] = Rs[9 * (size_t)a + i];
    for (int i = 0; i < 3; i++) m.t[i] = ts[3 * (size_t)a + i];
    m.pts = static_cast<const SiftPoint *>(sets[a].pts);
    m.n = sets[a].n;
    m.fixed = fixed ? fixed[a] : 0;
    if constexpr (NC == 9) {
      for (int i = 0; i < 2; i++) m.k[i] = dists ? dists[2 * (size_t)a + i] : 0.0;
      m.refine = refine ? refine[a] : 0;
    }
  }

  BaParams<NC> prm;
  prm.res = reinterpret_cast<BaResult *>(base + resAt);
  prm.flags = reinterpret_cast<unsigned int *>(base + flagsAt);
  prm.trace = reinterpret_cast<double *>(base + traceAt);
  prm.cams = reinterpret_cast<BaCam<NC> *>(base + camAt);
  prm.pts = reinterpret_cast<BaPt *>(base + ptAt);
  prm.cnt = reinterpret_cast<int *>(base + cntAt);
  prm.start = reinterpret_cast<int *>(base + startAt);
  prm.obs = reinterpret_cast<BaObs *>(base + obsAt);
  prm.J = reinterpret_cast<double *>(base + jAt);
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
  prm.errors = errors;
  prm.inlier = inlier;
  prm.thr2 = maxError * maxError;
  prm.tol2 = linearTol * linearTol;
  prm.numImages = C;
  prm.numTracks = T;
  prm.numMembers = M;
  prm.maxIterations = maxIterations;
  prm.maxLinear = maxLinearIterations;
  prm.loss = loss;
  prm.c2 = lossScale * lossScale;

  const int wave = coop_grid<bundle_kernel<NC, ROBUST>, BA_THREADS>("cs_bundle_adjust");
  if (wave < 0) return wave;
  const cudaStream_t st = c.stream;
  CS_CUDA(cudaMemsetAsync(base, 0, zeroEnd, st));
  if (C) CS_CUDA(cudaMemcpyAsync(prm.cams, cams, (size_t)C * sizeof(BaCam<NC>), cudaMemcpyHostToDevice, st));
  bundle_count_kernel<NC><<<std::max(idivup(T, BA_THREADS), 1), BA_THREADS, 0, st>>>(prm);
  count_launch();
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cub::DeviceScan::ExclusiveSum(base + tempAt, scanBytes, prm.cnt, prm.start, T + 1, st));
  bundle_fill_kernel<NC><<<std::max(idivup(std::max(T, M), BA_THREADS), 1), BA_THREADS, 0, st>>>(prm);
  count_launch();
  CS_CUDA(cudaGetLastError());
  if (M > 0)
    CS_CUDA(cub::DeviceRadixSort::SortPairs(base + tempAt, sortBytes, prm.keys, const_cast<int *>(prm.keysS), prm.vals,
                                            const_cast<int *>(prm.order), M, 0, bits, st));
  void *args[] = {&prm};
  CS_CUDA(cudaLaunchCooperativeKernel((const void *)bundle_kernel<NC, ROBUST>, dim3(wave), dim3(BA_THREADS), args, 0,
                                      st));
  count_launch();
  CS_CUDA(cudaMemcpyAsync(c.h_bundle.p, base + resAt, flagsAt - resAt, cudaMemcpyDeviceToHost, st));
  if (C) CS_CUDA(cudaMemcpyAsync(cams, prm.cams, (size_t)C * sizeof(BaCam<NC>), cudaMemcpyDeviceToHost, st));
  return 0;
}

}  // namespace

int bundle_camera_block(int numImages, const double *dists, const unsigned char *refine)
{
  for (int a = 0; a < numImages; a++)
    if ((refine && refine[a]) || (dists && (dists[2 * (size_t)a] != 0.0 || dists[2 * (size_t)a + 1] != 0.0)))
      return 9;
  return 6;
}

int bundle_enqueue(DeviceCtx &c, const cs_match_set *sets, int numImages, const double *Ks, const double *dists,
                   const unsigned char *refine, int loss, double lossScale, const double *Rs, const double *ts,
                   const unsigned char *fixed, const int *offsets, int numTracks, const int *members, int numMembers,
                   const unsigned char *use, double *points, int maxIterations, int maxLinearIterations,
                   double linearTol, double maxError, float *errors, unsigned char *inlier)
{
  const bool nine = bundle_camera_block(numImages, dists, refine) == 9;
#define CS_BUNDLE_RUN(NC, ROBUST)                                                                                      \
  bundle_run<NC, ROBUST>(c, sets, numImages, Ks, dists, refine, loss, lossScale, Rs, ts, fixed, offsets, numTracks,    \
                         members, numMembers, use, points, maxIterations, maxLinearIterations, linearTol, maxError,    \
                         errors, inlier)
  if (nine) return loss ? CS_BUNDLE_RUN(9, true) : CS_BUNDLE_RUN(9, false);
  return loss ? CS_BUNDLE_RUN(6, true) : CS_BUNDLE_RUN(6, false);
#undef CS_BUNDLE_RUN
}

namespace {

template <int NC>
int bundle_read(const DeviceCtx &c, int numImages, int maxIterations, double *K_out, double *dist_out, double *R_out,
                double *t_out, double cost[2], double *trace, long long stats[8])
{
  const size_t camAt = bundle_host_layout<NC>(numImages, maxIterations, nullptr);
  Layout H(256);
  H.take(sizeof(BaResult));
  const size_t trAt = H.take((size_t)maxIterations * 4 * sizeof(double));
  const BaResult *res = c.h_bundle.as<const BaResult>();
  const BaCam<NC> *cams = reinterpret_cast<const BaCam<NC> *>(c.h_bundle.as<const char>() + camAt);
  for (int a = 0; a < numImages; a++) {
    for (int i = 0; i < 9; i++) R_out[9 * (size_t)a + i] = cams[a].R[i];
    for (int i = 0; i < 3; i++) t_out[3 * (size_t)a + i] = cams[a].t[i];
    if constexpr (NC == 9) {
      if (K_out) {
        double *K = K_out + 9 * (size_t)a;
        for (int i = 0; i < 6; i++) K[i] = cams[a].K[i];
        K[6] = K[7] = 0.0;
        K[8] = 1.0;
      }
      if (dist_out)
        for (int i = 0; i < 2; i++) dist_out[2 * (size_t)a + i] = cams[a].k[i];
    }
  }
  if (cost) { cost[0] = res->cost[0]; cost[1] = res->cost[1]; }
  if (trace) memcpy(trace, c.h_bundle.as<const char>() + trAt, (size_t)maxIterations * 4 * sizeof(double));
  if (stats)
    for (int k = 0; k < 8; k++) stats[k] = (long long)res->stats[k];
  return (int)res->accepted;
}

}  // namespace

int bundle_result(const DeviceCtx &c, int nc, int numImages, int maxIterations, double *K_out, double *dist_out,
                  double *R_out, double *t_out, double cost[2], double *trace, long long stats[8])
{
  return nc == 9 ? bundle_read<9>(c, numImages, maxIterations, K_out, dist_out, R_out, t_out, cost, trace, stats)
                 : bundle_read<6>(c, numImages, maxIterations, K_out, dist_out, R_out, t_out, cost, trace, stats);
}

int undistort_enqueue(DeviceCtx &c, const cs_match_set *sets, int numImages, const double *Ks, const double *dists,
                      void *const *d_out)
{
  // one table in the bundle scratch: the images' K, k, records and first global indices
  const size_t bytes = (size_t)numImages * sizeof(UdImage);
  int r = c.bundle.grow(bytes);
  if (r < 0) return r;
  if ((r = c.h_bundle.grow(bytes)) < 0) return r;
  UdImage *imgs = c.h_bundle.as<UdImage>();
  long long total = 0;
  for (int a = 0; a < numImages; a++) {
    UdImage &m = imgs[a];
    memset(&m, 0, sizeof m);
    for (int i = 0; i < 6; i++) m.K[i] = Ks[9 * (size_t)a + i];
    for (int i = 0; i < 2; i++) m.k[i] = dists ? dists[2 * (size_t)a + i] : 0.0;
    m.in = static_cast<const SiftPoint *>(sets[a].pts);
    m.out = static_cast<SiftPoint *>(d_out[a]);
    m.first = total;
    m.n = sets[a].n;
    total += sets[a].n;
  }
  UdImage *d_imgs = c.bundle.as<UdImage>();
  CS_CUDA(cudaMemcpyAsync(d_imgs, imgs, bytes, cudaMemcpyHostToDevice, c.stream));
  undistort_kernel<<<(unsigned)((total + UD_THREADS - 1) / UD_THREADS), UD_THREADS, 0, c.stream>>>(d_imgs, numImages,
                                                                                                   total);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace cs
