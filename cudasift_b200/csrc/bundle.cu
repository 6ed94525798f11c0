// bundle.cu -- bundle adjustment of cameras and track points (cs_bundle_adjust).  The rules (used observations, gauge,
// residual, Levenberg-Marquardt, the Schur-complement solve, the outputs and the summation orders) are stated in
// cudasift_b200.h at cs_bundle_adjust; tests/bundle_oracle.py restates them in float64.
//
// Three counted launches, whatever the sizes and iteration counts:
//   1. bundle_count_kernel: per track, its used observations (0 when fewer than 2) and the integer statistics
//   2. (cub scan of the counts: each participating track's first observation)
//      bundle_fill_kernel: the used observations in track order, then member order, and a key (image) per observation
//   3. (cub stable radix sort of (image, observation): every camera's observations in observation order)
//      bundle_kernel: one cooperative launch runs the whole LM loop, phases separated by grid barriers
// Every floating-point sum has a fixed order that depends on the data only, not on the grid or on scheduling:
//   - per point: a thread sums its observations in observation order;
//   - per camera: the sorted observations are cut into tiles of BA_TILE; a warp sums a camera's piece of a tile
//     lane-strided, then by a fixed xor butterfly, and one lane per camera adds its pieces in ascending tile order;
//   - totals over points (the cost): a CTA sums a tile of 256 tracks by butterflies and its warps in order; over
//     cameras (the CG dot products): a warp sums a tile of 32 cameras by a butterfly; the tile partials are then added
//     by warp 0 of every CTA, lane-strided in ascending order and by a butterfly.
// No floating-point atomics.  Every branch around a grid barrier (the CG stop, the accept, the LM stop) is taken on
// values that every CTA computes from the same words, written before the barrier, by the same instructions in the same
// order, so every CTA takes the same path; every loop is bounded by maxIterations or maxLinearIterations.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <cooperative_groups.h>
#include <cub/cub.cuh>
#include <math_constants.h>

#include "common.cuh"
#include "vp_math.cuh"

namespace cg = cooperative_groups;

namespace cs {

namespace {

constexpr int BA_THREADS = 256;
constexpr int BA_WARPS = BA_THREADS / 32;
constexpr int BA_TILE = 256;         // sorted observations per camera tile
constexpr int BA_PV = 54;            // values of a camera piece: U (21), g (6), W V*^-1 g_p (6), the Schur term (21)
constexpr int BA_JD = 20;            // doubles per observation: J_c (2 x 6), J_p (2 x 3), r (2)
// Slots per camera tile partial.  p.S p has a slot of its own: CG phase G writes r.r and r.z with no grid barrier after
// the totals of p.S p are read, so they may not share a slot.
constexpr int BA_CP = 3;

// A used observation: its track, image, member and pixel position.
struct BaObs {
  int k, a, m, pad;
  float x, y;
};

// A camera: the input, the state of the LM loop and its sorted observations [start, end).
struct BaCam {
  double K[6];                       // K[0..5] of the row-major K (K[3] unused)
  double R[9], t[3];                 // current
  double Rc[9], tc[3];               // candidate
  double P[12];                      // K [R | t] of the final parameters (outputs)
  double U[21];                      // U* (damped), upper triangle row by row; held rows and columns are identity
  double L[21];                      // Cholesky factor of the preconditioner block, lower triangle row by row
  double x[6], r[6], z[6], p[6], q[6];
  const SiftPoint *pts;
  int n, fixed, mask, start, end, pad;
};

static_assert(sizeof(BaCam) == 944, "the header states the per-image scratch");

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

struct BaParams {
  BaCam *cams;
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
  double *J;                         // [numMembers][BA_JD]
  int *keys, *vals;                  // [numMembers]: image and observation, sorted in keysS / order
  const int *keysS, *order;
  double *pieces;                    // [tiles + numImages][BA_PV]
  double *camPart;                   // [ceil(numImages / 32)][BA_CP]: r.r (or b~.b~), r.z, p.S p
  double *ptPart;                    // [ceil(numTracks / 256)][2]
  unsigned int *flags;               // [maxIterations]: a Cholesky pivot failed in iteration it
  double *trace;                     // [maxIterations][4]
  BaResult *res;
  double thr2, tol2;
  int numImages, numTracks, numMembers, maxIterations, maxLinear;
};

// ---- small dense helpers (row-major full matrices in registers) ----------------------------------------------------

// Cholesky of the symmetric A (N x N); false when a pivot is not > 0 or not finite.  L is lower, packed row by row.
template <int N>
__device__ __forceinline__ bool ba_chol(const double (&A)[N][N], double *L)
{
  double F[N][N];
#pragma unroll
  for (int j = 0; j < N; j++) {
    double d = A[j][j];
#pragma unroll
    for (int q = 0; q < j; q++) d -= F[j][q] * F[j][q];
    if (!(d > 0.0) || !isfinite(d)) return false;
    F[j][j] = sqrt(d);
#pragma unroll
    for (int i = j + 1; i < N; i++) {
      double e = A[i][j];
#pragma unroll
      for (int q = 0; q < j; q++) e -= F[i][q] * F[j][q];
      F[i][j] = e / F[j][j];
    }
  }
  int k = 0;
#pragma unroll
  for (int i = 0; i < N; i++)
#pragma unroll
    for (int j = 0; j <= i; j++) L[k++] = F[i][j];
  return true;
}

// x = A^-1 b from the packed factor of ba_chol (forward, then backward substitution)
template <int N>
__device__ __forceinline__ void ba_chol_solve(const double *L, const double (&b)[N], double (&x)[N])
{
  double z[N];
#pragma unroll
  for (int i = 0; i < N; i++) {
    double e = b[i];
#pragma unroll
    for (int q = 0; q < i; q++) e -= L[i * (i + 1) / 2 + q] * z[q];
    z[i] = e / L[i * (i + 1) / 2 + i];
  }
#pragma unroll
  for (int i = N - 1; i >= 0; i--) {
    double e = z[i];
#pragma unroll
    for (int q = i + 1; q < N; q++) e -= L[q * (q + 1) / 2 + i] * x[q];
    x[i] = e / L[i * (i + 1) / 2 + i];
  }
}

// the damped diagonal entry d + lambda clamp(d, 1e-6, 1e32)
__device__ __forceinline__ double ba_damp(double d, double lam) { return d + lam * fmin(fmax(d, 1e-6), 1e32); }

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

// ---- setup kernels --------------------------------------------------------------------------------------------------

// The used observations of track k (through f(m, a, x, y)); -1 for a malformed track.
template <class F>
__device__ __forceinline__ int ba_used(const BaParams &p, int k, int &invalid, F &&f)
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
    const BaCam &c = p.cams[af.x];
    if (!(ba_depth(c.R, c.t, X) > 0.0)) continue;
    f(m, af.x, x, y, used);
    used++;
  }
  return used;
}

__global__ void __launch_bounds__(BA_THREADS) bundle_count_kernel(BaParams p)
{
  const int k = blockIdx.x * BA_THREADS + threadIdx.x;
  if (k == 0) p.cnt[p.numTracks] = 0;
  if (k >= p.numTracks) return;
  int invalid = 0;
  const int used = ba_used(p, k, invalid, [](int, int, float, float, int) {});
  unsigned long long *st = p.res->stats;
  if (used < 0) {
    atomicAdd(&st[1], 1ull);
    p.cnt[k] = 0;
    return;
  }
  atomicAdd(&st[0], 1ull);
  if (invalid) atomicAdd(&st[2], (unsigned long long)invalid);
  p.cnt[k] = used >= 2 ? used : 0;
  if (used >= 2) {
    atomicAdd(&st[3], (unsigned long long)used);
    atomicAdd(&st[4], 1ull);
  }
}

__global__ void __launch_bounds__(BA_THREADS) bundle_fill_kernel(BaParams p)
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

// The K sums of n tile partials (part[tile * stride + j]): warp 0 adds them lane-strided in ascending order, then by a
// fixed xor butterfly; every thread of the CTA receives them.  Every CTA reads the partials after the barrier that
// follows their writes, so a slot read here must not be written again before the next grid barrier.
template <int K>
__device__ __forceinline__ void ba_totals(const double *part, int n, int stride, double (&out)[K])
{
  __shared__ double s_tot[K];
  if (threadIdx.x < 32) {
    double v[K];
#pragma unroll
    for (int j = 0; j < K; j++) v[j] = 0.0;
    for (int i = (int)threadIdx.x; i < n; i += 32)
#pragma unroll
      for (int j = 0; j < K; j++) v[j] += part[(size_t)i * stride + j];
    vp_warp_sum(v);
    if (threadIdx.x == 0)
#pragma unroll
      for (int j = 0; j < K; j++) s_tot[j] = v[j];
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < K; j++) out[j] = s_tot[j];
  __syncthreads();                                           // s_tot is read before the next call writes it
}

// A CTA's tile partial of K values (one per thread): warp butterflies, then thread 0 adds the warps in order.
template <int K>
__device__ __forceinline__ void ba_cta_partial(double (&v)[K], double *out)
{
  __shared__ double s_w[BA_WARPS][K];
  vp_warp_sum(v);
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int j = 0; j < K; j++) s_w[threadIdx.x >> 5][j] = v[j];
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int j = 0; j < K; j++) {
      double s = s_w[0][j];
      for (int w = 1; w < BA_WARPS; w++) s += s_w[w][j];
      out[j] = s;
    }
  __syncthreads();
}

// A warp's tile partial of K values (one per lane, a lane per camera): a butterfly, lane 0 writes.
template <int K>
__device__ __forceinline__ void ba_warp_partial(double (&v)[K], double *out)
{
  vp_warp_sum(v);
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int j = 0; j < K; j++) out[j] = v[j];
}

// The camera pieces of NV values per observation (f(o, a, v)) at offset OFF: a warp per tile of BA_TILE sorted
// observations, each camera's piece summed lane-strided and by a butterfly, stored at piece index tile + camera
// (unique: a camera's tiles follow the previous camera's last one).
template <int NV, int OFF, class F>
__device__ __forceinline__ void ba_pieces(const BaParams &p, int N, F &&f)
{
  const int lane = threadIdx.x & 31;
  const int numWarps = (int)gridDim.x * BA_WARPS, numTiles = (N + BA_TILE - 1) / BA_TILE;
  for (int t = (int)((blockIdx.x * BA_THREADS + threadIdx.x) >> 5); t < numTiles; t += numWarps) {
    const int t1 = min(N, (t + 1) * BA_TILE);
    for (int s = t * BA_TILE; s < t1;) {
      const int a = p.keysS[s];
      const int e = min(t1, p.cams[a].end);
      double acc[NV];
#pragma unroll
      for (int j = 0; j < NV; j++) acc[j] = 0.0;
      for (int i = s + lane; i < e; i += 32) {
        double v[NV];
        f(p.order[i], a, v);
#pragma unroll
        for (int j = 0; j < NV; j++) acc[j] += v[j];
      }
      vp_warp_sum(acc);
      if (lane == 0)
#pragma unroll
        for (int j = 0; j < NV; j++) p.pieces[(size_t)(t + a) * BA_PV + OFF + j] = acc[j];
      s = e;
    }
  }
}

// The sum of camera c's pieces (NV values at OFF) in ascending tile order.
template <int NV, int OFF>
__device__ __forceinline__ void ba_gather(const BaParams &p, int a, const BaCam &c, double (&v)[NV])
{
#pragma unroll
  for (int j = 0; j < NV; j++) v[j] = 0.0;
  if (c.end > c.start)
    for (int t = c.start / BA_TILE; t <= (c.end - 1) / BA_TILE; t++)
#pragma unroll
      for (int j = 0; j < NV; j++) v[j] += p.pieces[(size_t)(t + a) * BA_PV + OFF + j];
}

// J_c^T (J_p y) of observation o (6 values)
__device__ __forceinline__ void ba_wy(const double *J, const double *y, double *v)
{
  const double s0 = J[12] * y[0] + J[13] * y[1] + J[14] * y[2], s1 = J[15] * y[0] + J[16] * y[1] + J[17] * y[2];
#pragma unroll
  for (int i = 0; i < 6; i++) v[i] = J[i] * s0 + J[6 + i] * s1;
}

// J_p^T (J_c x), accumulated into h (3 values)
__device__ __forceinline__ void ba_wtx(const double *J, const double *x, double (&h)[3])
{
  double s0 = 0.0, s1 = 0.0;
#pragma unroll
  for (int i = 0; i < 6; i++) { s0 += J[i] * x[i]; s1 += J[6 + i] * x[i]; }
#pragma unroll
  for (int j = 0; j < 3; j++) h[j] += J[12 + j] * s0 + J[15 + j] * s1;
}

// the packed upper-triangle index of (i, j), i <= j, of a 6 x 6 matrix
__device__ __forceinline__ int ba_up6(int i, int j) { return i * 6 - i * (i - 1) / 2 + (j - i); }

// Per participating track (a thread each, tiles of 256 tracks per CTA): f(k, s, e) returns K values for the tile
// partials at part (or nothing with K == 0).
template <int K, class F>
__device__ __forceinline__ void ba_per_point(const BaParams &p, double *part, F &&f)
{
  for (int base = (int)blockIdx.x * BA_THREADS; base < p.numTracks; base += (int)gridDim.x * BA_THREADS) {
    const int k = base + (int)threadIdx.x;
    double v[K > 0 ? K : 1];
#pragma unroll
    for (int j = 0; j < (K > 0 ? K : 1); j++) v[j] = 0.0;
    if (k < p.numTracks) {
      const int s = p.start[k], e = p.start[k + 1];
      if (e > s) f(k, s, e, v);
    }
    if constexpr (K > 0) ba_cta_partial<K>(v, part + (size_t)(base / BA_THREADS) * K);
  }
}

// Linearise every observation of track k at the current parameters (or the candidate ones); returns its cost.
__device__ __forceinline__ double ba_relinearise(const BaParams &p, int k, int s, int e, bool cand)
{
  const BaPt &pt = p.pts[k];
  const double X[3] = {cand ? pt.Xc[0] : pt.X[0], cand ? pt.Xc[1] : pt.X[1], cand ? pt.Xc[2] : pt.X[2]};
  double cost = 0.0;
  for (int o = s; o < e; o++) {
    const BaObs ob = p.obs[o];
    const BaCam &c = p.cams[ob.a];
    double r[2];
    ba_linearise(c.K, cand ? c.Rc : c.R, cand ? c.tc : c.t, X, ob.x, ob.y, r, p.J + (size_t)o * BA_JD);
    cost += r[0] * r[0] + r[1] * r[1];
  }
  return cost;
}

__global__ void __launch_bounds__(BA_THREADS) bundle_kernel(BaParams p)
{
  cg::grid_group grid = cg::this_grid();
  const int tid = (int)(blockIdx.x * BA_THREADS + threadIdx.x), nthreads = (int)gridDim.x * BA_THREADS;
  const int lane = (int)threadIdx.x & 31;
  const int warpG = tid >> 5, numWarps = nthreads >> 5;
  const int C = p.numImages, N = p.start[p.numTracks];
  const int camTiles = (C + 31) / 32, ptTiles = (p.numTracks + BA_THREADS - 1) / BA_THREADS;

  // 0. every camera's sorted range, its free components; the linearisation at the input and its cost
  for (int i = tid; i < N; i += nthreads) {
    const int a = p.keysS[i];
    if (i == 0 || p.keysS[i - 1] != a) p.cams[a].start = i;
    if (i == N - 1 || p.keysS[i + 1] != a) p.cams[a].end = i + 1;
  }
  grid.sync();
  for (int a = tid; a < C; a += nthreads) {
    BaCam &c = p.cams[a];
    c.mask = c.end > c.start ? ba_free_mask(c.fixed) : 0;
    if (c.mask) atomicAdd(&p.res->stats[5], (unsigned long long)__popc(c.mask));
  }
  ba_per_point<1>(p, p.ptPart, [&](int k, int s, int e, double *v) { v[0] = ba_relinearise(p, k, s, e, false); });
  grid.sync();
  double cost;
  {
    double t[1];
    ba_totals<1>(p.ptPart, ptTiles, 1, t);
    cost = t[0];
  }
  const double cost0 = cost;
  double lam = 1e-3;
  unsigned long long accepted = 0, lmIters = 0, cgTotal = 0;

  for (int it = 0; it < p.maxIterations && N > 0; it++) {
    lmIters++;
    // A. per point: V* (damped) by Cholesky, g_p = J_p^T r, q = V*^-1 g_p
    ba_per_point<0>(p, nullptr, [&](int k, int s, int e, double *) {
      double V[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, g[3] = {0, 0, 0};
      for (int o = s; o < e; o++) {
        const double *J = p.J + (size_t)o * BA_JD;
#pragma unroll
        for (int q = 0; q < 2; q++) {
          const double *jp = J + 12 + 3 * q, r = J[18 + q];
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
        V[i][i] = ba_damp(V[i][i], lam);
#pragma unroll
        for (int j = 0; j < i; j++) V[i][j] = V[j][i];
      }
      BaPt &pt = p.pts[k];
      if (!ba_chol<3>(V, pt.L)) { atomicOr(&p.flags[it], 1u); return; }
      double q[3];
      ba_chol_solve<3>(pt.L, g, q);
#pragma unroll
      for (int i = 0; i < 3; i++) { pt.g[i] = g[i]; pt.q[i] = q[i]; }
    });
    grid.sync();
    unsigned int fail = *(volatile unsigned int *)&p.flags[it];

    // B. the camera pieces: U, g_c, W q and the Schur term W_o V*^-1 W_ak^T (W_ak: the track's observations in image a)
    if (!fail) {
      ba_pieces<21, 0>(p, N, [&](int o, int, double *v) {
        const double *J = p.J + (size_t)o * BA_JD;
        int n = 0;
#pragma unroll
        for (int i = 0; i < 6; i++)
#pragma unroll
          for (int j = i; j < 6; j++) v[n++] = J[i] * J[j] + J[6 + i] * J[6 + j];
      });
      ba_pieces<12, 21>(p, N, [&](int o, int, double *v) {
        const double *J = p.J + (size_t)o * BA_JD;
        const double *q = p.pts[p.obs[o].k].q;
#pragma unroll
        for (int i = 0; i < 6; i++) v[i] = J[i] * J[18] + J[6 + i] * J[19];
        ba_wy(J, q, v + 6);
      });
      ba_pieces<21, 33>(p, N, [&](int o, int a, double *v) {
        const double *J = p.J + (size_t)o * BA_JD;
        const int k = p.obs[o].k;
        double Wo[6][3], Wa[6][3], Y[6][3];
#pragma unroll
        for (int i = 0; i < 6; i++)
#pragma unroll
          for (int j = 0; j < 3; j++) { Wo[i][j] = J[i] * J[12 + j] + J[6 + i] * J[15 + j]; Wa[i][j] = 0.0; }
        for (int u = p.start[k]; u < p.start[k + 1]; u++) {
          if (p.obs[u].a != a) continue;
          const double *Ju = p.J + (size_t)u * BA_JD;
#pragma unroll
          for (int i = 0; i < 6; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) Wa[i][j] += Ju[i] * Ju[12 + j] + Ju[6 + i] * Ju[15 + j];
        }
        const double *L = p.pts[k].L;
#pragma unroll
        for (int i = 0; i < 6; i++) ba_chol_solve<3>(L, Wa[i], Y[i]);
        int n = 0;
#pragma unroll
        for (int i = 0; i < 6; i++)
#pragma unroll
          for (int j = i; j < 6; j++) v[n++] = Wo[i][0] * Y[j][0] + Wo[i][1] * Y[j][1] + Wo[i][2] * Y[j][2];
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
          BaCam &c = p.cams[a];
          double U[21], G[12], T[21];
          ba_gather<21, 0>(p, a, c, U);
          ba_gather<12, 21>(p, a, c, G);
          ba_gather<21, 33>(p, a, c, T);
          double Us[6][6], M[6][6];
#pragma unroll
          for (int i = 0; i < 6; i++)
#pragma unroll
            for (int j = i; j < 6; j++) {
              const bool fr = ((c.mask >> i) & 1) && ((c.mask >> j) & 1);
              double u = U[ba_up6(i, j)];
              if (i == j) u = ba_damp(u, lam);
              Us[i][j] = Us[j][i] = fr ? u : (i == j ? 1.0 : 0.0);
              M[i][j] = M[j][i] = fr ? u - T[ba_up6(i, j)] : (i == j ? 1.0 : 0.0);
            }
#pragma unroll
          for (int i = 0; i < 6; i++)
#pragma unroll
            for (int j = i; j < 6; j++) c.U[ba_up6(i, j)] = Us[i][j];
          if (!ba_chol<6>(M, c.L)) {
            atomicOr(&p.flags[it], 1u);
          } else {
            double r[6], z[6];
#pragma unroll
            for (int i = 0; i < 6; i++) r[i] = ((c.mask >> i) & 1) ? -G[i] + G[6 + i] : 0.0;
            ba_chol_solve<6>(c.L, r, z);
#pragma unroll
            for (int i = 0; i < 6; i++) {
              c.x[i] = 0.0; c.r[i] = r[i]; c.z[i] = z[i]; c.p[i] = 0.0;
              d[0] += r[i] * r[i];
              d[1] += r[i] * z[i];
            }
          }
        }
        ba_warp_partial<2>(d, p.camPart + BA_CP * (size_t)w);
      }
    grid.sync();
    fail = *(volatile unsigned int *)&p.flags[it];

    // D-G. preconditioned CG on S dc = b~ from dc = 0
    int cgIt = 0;
    if (!fail) {
      double t2[2];
      ba_totals<2>(p.camPart, camTiles, BA_CP, t2);
      const double thr = p.tol2 * t2[0];
      double rr = t2[0], rz = t2[1], beta = 0.0;
      while (cgIt < p.maxLinear && !(rr <= thr)) {
        // D. per point: y = V*^-1 W^T p, with p = z + beta p_old of each camera
        ba_per_point<0>(p, nullptr, [&](int k, int s, int e, double *) {
          double h[3] = {0.0, 0.0, 0.0};
          for (int o = s; o < e; o++) {
            const BaCam &c = p.cams[p.obs[o].a];
            double pe[6];
#pragma unroll
            for (int i = 0; i < 6; i++) pe[i] = fma(beta, c.p[i], c.z[i]);
            ba_wtx(p.J + (size_t)o * BA_JD, pe, h);
          }
          BaPt &pt = p.pts[k];
          double y[3];
          ba_chol_solve<3>(pt.L, h, y);
#pragma unroll
          for (int i = 0; i < 3; i++) pt.y[i] = y[i];
        });
        grid.sync();
        // E. the camera pieces of W y
        ba_pieces<6, 0>(p, N, [&](int o, int, double *v) {
          ba_wy(p.J + (size_t)o * BA_JD, p.pts[p.obs[o].k].y, v);
        });
        grid.sync();
        // F. per camera: p = z + beta p_old, q = S p = U* p - W y (held components 0); the partials of p.q
        for (int w = warpG; w < camTiles; w += numWarps) {
          const int a = w * 32 + lane;
          double d[1] = {0.0};
          if (a < C) {
            BaCam &c = p.cams[a];
            double Wy[6], pn[6];
            ba_gather<6, 0>(p, a, c, Wy);
#pragma unroll
            for (int i = 0; i < 6; i++) pn[i] = fma(beta, c.p[i], c.z[i]);
#pragma unroll
            for (int i = 0; i < 6; i++) {
              double s = 0.0;
#pragma unroll
              for (int j = 0; j < 6; j++) s += c.U[ba_up6(min(i, j), max(i, j))] * pn[j];
              const double q = ((c.mask >> i) & 1) ? s - Wy[i] : 0.0;
              c.p[i] = pn[i];
              c.q[i] = q;
              d[0] += pn[i] * q;
            }
          }
          ba_warp_partial<1>(d, p.camPart + BA_CP * (size_t)w + 2);
        }
        grid.sync();
        double pq[1];
        ba_totals<1>(p.camPart + 2, camTiles, BA_CP, pq);
        if (!(pq[0] > 0.0)) break;
        const double alpha = rz / pq[0];
        // G. per camera: x += alpha p, r -= alpha q, z = M^-1 r; the partials of r.r and r.z
        for (int w = warpG; w < camTiles; w += numWarps) {
          const int a = w * 32 + lane;
          double d[2] = {0.0, 0.0};
          if (a < C) {
            BaCam &c = p.cams[a];
            double r[6], z[6];
#pragma unroll
            for (int i = 0; i < 6; i++) {
              c.x[i] = fma(alpha, c.p[i], c.x[i]);
              r[i] = fma(-alpha, c.q[i], c.r[i]);
              c.r[i] = r[i];
            }
            ba_chol_solve<6>(c.L, r, z);
#pragma unroll
            for (int i = 0; i < 6; i++) {
              c.z[i] = z[i];
              d[0] += r[i] * r[i];
              d[1] += r[i] * z[i];
            }
          }
          ba_warp_partial<2>(d, p.camPart + BA_CP * (size_t)w);
        }
        cgIt++;
        grid.sync();
        ba_totals<2>(p.camPart, camTiles, BA_CP, t2);
        rr = t2[0];
        beta = t2[1] / rz;
        rz = t2[1];
      }
    }
    cgTotal += cgIt;

    // H. back-substitution dp = V*^-1 (-g_p - W^T dc) and the candidate points; the candidate cameras
    double cand[2] = {CUDART_NAN, 0.0};
    if (!fail) {
      ba_per_point<0>(p, nullptr, [&](int k, int s, int e, double *) {
        BaPt &pt = p.pts[k];
        double h[3] = {0.0, 0.0, 0.0}, dp[3];
        for (int o = s; o < e; o++) ba_wtx(p.J + (size_t)o * BA_JD, p.cams[p.obs[o].a].x, h);
#pragma unroll
        for (int i = 0; i < 3; i++) h[i] = -pt.g[i] - h[i];
        ba_chol_solve<3>(pt.L, h, dp);
#pragma unroll
        for (int i = 0; i < 3; i++) pt.Xc[i] = pt.X[i] + dp[i];
      });
      for (int a = tid; a < C; a += nthreads) {
        BaCam &c = p.cams[a];
        if (!c.mask) {
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
      // I. the candidate's cost and its observations behind a camera
      ba_per_point<2>(p, p.ptPart, [&](int k, int s, int e, double *v) {
        const BaPt &pt = p.pts[k];
        const double X[3] = {pt.Xc[0], pt.Xc[1], pt.Xc[2]};
        for (int o = s; o < e; o++) {
          const BaObs ob = p.obs[o];
          const BaCam &c = p.cams[ob.a];
          double r[2];
          const double z = ba_linearise(c.K, c.Rc, c.tc, X, ob.x, ob.y, r, nullptr);
          v[0] += r[0] * r[0] + r[1] * r[1];
          if (!(z > 0.0)) v[1] += 1.0;
        }
      });
      grid.sync();
      ba_totals<2>(p.ptPart, ptTiles, 2, cand);
    }

    // J. accept or reject
    const bool accept = !fail && cand[1] == 0.0 && cand[0] < cost;
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
        BaCam &c = p.cams[a];
#pragma unroll
        for (int i = 0; i < 9; i++) c.R[i] = c.Rc[i];
#pragma unroll
        for (int i = 0; i < 3; i++) c.t[i] = c.tc[i];
      }
      ba_per_point<0>(p, nullptr, [&](int k, int s, int e, double *) {
        ba_relinearise(p, k, s, e, true);
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
    BaCam &c = p.cams[a];
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
      if (tr_member(p.cams, C, af, x, y) && has) tr_reproject(p.cams[af.x].P, X, x, y, p.thr2, err, in);
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

// One resident wave of the cooperative kernel; CS_E_CUDA without cooperative launch.
int bundle_grid()
{
  int dev = 0, coop = 0;
  CS_CUDA(cudaGetDevice(&dev));
  CS_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  if (!coop) {
    set_error("cs_bundle_adjust: device %d does not support cooperative launches", dev);
    return CS_E_CUDA;
  }
  return resident_grid<bundle_kernel, BA_THREADS>();
}

}  // namespace

int bundle_enqueue(DeviceCtx &c, const cs_match_set *sets, int numImages, const double *Ks, const double *Rs,
                   const double *ts, const unsigned char *fixed, const int *offsets, int numTracks, const int *members,
                   int numMembers, const unsigned char *use, double *points, int maxIterations, int maxLinearIterations,
                   double linearTol, double maxError, float *errors, unsigned char *inlier)
{
  const int M = numMembers, T = numTracks, C = numImages;
  const int tiles = (M + BA_TILE - 1) / BA_TILE;
  int bits = 1;
  while (bits < 31 && (1ll << bits) <= (long long)C) bits++;        // every key, the sentinel C included, is < 2^bits
  size_t scanBytes = 0, sortBytes = 0;
  CS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scanBytes, (int *)nullptr, (int *)nullptr, T + 1, c.stream));
  CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sortBytes, (int *)nullptr, (int *)nullptr, (int *)nullptr,
                                          (int *)nullptr, std::max(M, 1), 0, bits, c.stream));

  // device scratch (header: cs_bundle_adjust)
  Layout L(256);
  const size_t resAt = L.take(sizeof(BaResult)), traceAt = L.take((size_t)maxIterations * 4 * sizeof(double));
  const size_t flagsAt = L.take((size_t)maxIterations * sizeof(unsigned int)), zeroEnd = L.bytes;
  const size_t camAt = L.take((size_t)C * sizeof(BaCam)), ptAt = L.take((size_t)T * sizeof(BaPt));
  const size_t cntAt = L.take(((size_t)T + 1) * sizeof(int)), startAt = L.take(((size_t)T + 1) * sizeof(int));
  const size_t obsAt = L.take((size_t)M * sizeof(BaObs)), jAt = L.take((size_t)M * BA_JD * sizeof(double));
  const size_t keysAt = L.take((size_t)M * sizeof(int)), valsAt = L.take((size_t)M * sizeof(int));
  const size_t keysSAt = L.take((size_t)M * sizeof(int)), orderAt = L.take((size_t)M * sizeof(int));
  const size_t piecesAt = L.take(((size_t)tiles + C) * BA_PV * sizeof(double));
  const size_t camPartAt = L.take((size_t)idivup(C, 32) * BA_CP * sizeof(double));
  const size_t ptPartAt = L.take((size_t)idivup(T, BA_THREADS) * 2 * sizeof(double));
  const size_t tempAt = L.take(std::max(scanBytes, sortBytes));
  int r = c.bundle.grow(L.bytes);
  if (r < 0) return r;
  char *base = c.bundle.as<char>();

  // pinned: the result words and the trace (copied back), then the camera table (uploaded, then copied back)
  // (the same offsets as the device's result words and trace, so that one copy brings both back)
  Layout H(256);
  H.take(sizeof(BaResult));
  H.take((size_t)maxIterations * 4 * sizeof(double));
  const size_t hCamAt = H.take((size_t)C * sizeof(BaCam));
  if ((r = c.h_bundle.grow(H.bytes)) < 0) return r;
  BaCam *cams = reinterpret_cast<BaCam *>(c.h_bundle.as<char>() + hCamAt);
  for (int a = 0; a < C; a++) {
    BaCam &m = cams[a];
    memset(&m, 0, sizeof m);
    for (int i = 0; i < 6; i++) m.K[i] = Ks[9 * (size_t)a + i];
    for (int i = 0; i < 9; i++) m.R[i] = Rs[9 * (size_t)a + i];
    for (int i = 0; i < 3; i++) m.t[i] = ts[3 * (size_t)a + i];
    m.pts = static_cast<const SiftPoint *>(sets[a].pts);
    m.n = sets[a].n;
    m.fixed = fixed ? fixed[a] : 0;
  }

  BaParams prm;
  prm.res = reinterpret_cast<BaResult *>(base + resAt);
  prm.flags = reinterpret_cast<unsigned int *>(base + flagsAt);
  prm.trace = reinterpret_cast<double *>(base + traceAt);
  prm.cams = reinterpret_cast<BaCam *>(base + camAt);
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

  const int wave = bundle_grid();
  if (wave < 0) return wave;
  const cudaStream_t st = c.stream;
  CS_CUDA(cudaMemsetAsync(base, 0, zeroEnd, st));
  if (C) CS_CUDA(cudaMemcpyAsync(prm.cams, cams, (size_t)C * sizeof(BaCam), cudaMemcpyHostToDevice, st));
  bundle_count_kernel<<<std::max(idivup(T, BA_THREADS), 1), BA_THREADS, 0, st>>>(prm);
  count_launch();
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cub::DeviceScan::ExclusiveSum(base + tempAt, scanBytes, prm.cnt, prm.start, T + 1, st));
  bundle_fill_kernel<<<std::max(idivup(std::max(T, M), BA_THREADS), 1), BA_THREADS, 0, st>>>(prm);
  count_launch();
  CS_CUDA(cudaGetLastError());
  if (M > 0)
    CS_CUDA(cub::DeviceRadixSort::SortPairs(base + tempAt, sortBytes, prm.keys, const_cast<int *>(prm.keysS), prm.vals,
                                            const_cast<int *>(prm.order), M, 0, bits, st));
  void *args[] = {&prm};
  CS_CUDA(cudaLaunchCooperativeKernel((const void *)bundle_kernel, dim3(wave), dim3(BA_THREADS), args, 0, st));
  count_launch();
  CS_CUDA(cudaMemcpyAsync(c.h_bundle.p, base + resAt, flagsAt - resAt, cudaMemcpyDeviceToHost, st));
  if (C) CS_CUDA(cudaMemcpyAsync(cams, prm.cams, (size_t)C * sizeof(BaCam), cudaMemcpyDeviceToHost, st));
  return 0;
}

int bundle_result(const DeviceCtx &c, int numImages, int maxIterations, double *R_out, double *t_out, double cost[2],
                  double *trace, long long stats[8])
{
  Layout H(256);
  H.take(sizeof(BaResult));
  const size_t traceAt = H.take((size_t)maxIterations * 4 * sizeof(double)), camAt = H.take(0);
  const BaResult *res = c.h_bundle.as<const BaResult>();
  const BaCam *cams = reinterpret_cast<const BaCam *>(c.h_bundle.as<const char>() + camAt);
  for (int a = 0; a < numImages; a++) {
    for (int i = 0; i < 9; i++) R_out[9 * (size_t)a + i] = cams[a].R[i];
    for (int i = 0; i < 3; i++) t_out[3 * (size_t)a + i] = cams[a].t[i];
  }
  if (cost) { cost[0] = res->cost[0]; cost[1] = res->cost[1]; }
  if (trace) memcpy(trace, c.h_bundle.as<const char>() + traceAt, (size_t)maxIterations * 4 * sizeof(double));
  if (stats)
    for (int k = 0; k < 8; k++) stats[k] = (long long)res->stats[k];
  return (int)res->accepted;
}

}  // namespace cs
