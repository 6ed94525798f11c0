// vp_math.cuh -- the FP64 helpers that geometric verification (verify.cu), triangulation (triangulate.cu), absolute
// pose (pose.cu), bundle adjustment (bundle.cu) and the vocabulary's start draws (vocab.cu) share: the counter-based
// generator and sampler, the cyclic Jacobi eigen-decomposition, the calibrated coordinates of a pinhole K, the fixed
// xor butterflies (a sum over K doubles, a max over a u64 key), the Rodrigues rotation and the left rotation update,
// the member rule of a track, and the reprojection inlier rule and per-observation output; the small Cholesky and its
// solve, the Levenberg-Marquardt damping term and the robust losses of bundle adjustment and global positioning
// (globalpos.cu); and the hypothesis prologue and slot arg-max of the two batched RANSAC calls (verify.cu, pose.cu).
// tests/verify_oracle.py and tests/triangulate_oracle.py restate the rules in float64.
#pragma once

#include <cmath>
#include <math_constants.h>

namespace cs {

__host__ __device__ inline unsigned long long vp_splitmix64(unsigned long long z)
{
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// Symmetric eigen-decomposition by cyclic Jacobi: a becomes diagonal, the columns of v are the eigenvectors.
template <int N>
__host__ __device__ inline void vp_jacobi(double (&a)[N][N], double (&v)[N][N])
{
  double tot = 0.0;
  for (int p = 0; p < N; p++)
    for (int q = 0; q < N; q++) { v[p][q] = p == q ? 1.0 : 0.0; tot += a[p][q] * a[p][q]; }
  for (int sweep = 0; sweep < 30; sweep++) {
    double off = 0.0;
    for (int p = 0; p < N; p++)
      for (int q = p + 1; q < N; q++) off += a[p][q] * a[p][q];
    if (!(off > 1e-32 * tot)) break;
    for (int p = 0; p < N; p++)
      for (int q = p + 1; q < N; q++) {
        // after three sweeps an element too small to change either diagonal entry is set to zero (Numerical Recipes'
        // rule), so that the sweeps end instead of running against rounding
        const double g = 100.0 * fabs(a[p][q]);
        if (sweep > 2 && fabs(a[p][p]) + g == fabs(a[p][p]) && fabs(a[q][q]) + g == fabs(a[q][q])) {
          a[p][q] = a[q][p] = 0.0;
          continue;
        }
        if (a[p][q] == 0.0) continue;
        const double th = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
        const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < N; k++) {
          const double kp = a[k][p], kq = a[k][q];
          a[k][p] = c * kp - s * kq; a[k][q] = s * kp + c * kq;
        }
        for (int k = 0; k < N; k++) {
          const double pk = a[p][k], qk = a[q][k];
          a[p][k] = c * pk - s * qk; a[q][k] = s * pk + c * qk;
        }
        for (int k = 0; k < N; k++) {
          const double kp = v[k][p], kq = v[k][q];
          v[k][p] = c * kp - s * kq; v[k][q] = s * kp + c * kq;
        }
      }
  }
}

// calibrated coordinates x^ = K^-1 (x, y, 1) of an upper-triangular K: y^ = (y - K[5]) / K[4], x^ = (x - K[2] - K[1] y^) / K[0]
__host__ __device__ inline void vp_calibrate(const double *K, double x, double y, double &cx, double &cy)
{
  cy = (y - K[5]) / K[4];
  cx = (x - K[2] - K[1] * cy) / K[0];
}

#define VP_MAX_DRAWS 64

// The k distinct indices of sample smp into the n valid items (the rule of cs_verify_pairs); false when n < K or after
// 64 draws.
template <int K>
__device__ bool vp_draw(unsigned long long seed, int smp, int n, int (&idx)[K])
{
  if (n < K) return false;
  int got = 0;
  for (int d = 0; d < VP_MAX_DRAWS && got < K; d++) {
    const unsigned long long x = vp_splitmix64(seed + 0x9E3779B97F4A7C15ull * (((unsigned long long)smp << 8) | (unsigned)d));
    const int i = (int)(((x >> 32) * (unsigned long long)n) >> 32);
    bool dup = false;
#pragma unroll
    for (int j = 0; j < K; j++) dup |= (j < got && idx[j] == i);
    if (dup) continue;
#pragma unroll
    for (int j = 0; j < K; j++) if (j == got) idx[j] = i;
    got++;
  }
  return got == K;
}

// The prologue of a RANSAC hypothesis kernel (idivup(numLoops, T) CTAs of T threads per job, one thread per sample):
// the thread's job j and sample smp, then the sample's PER slots of D doubles NaN-filled (an empty slot) with zero
// counts.  slots and counts are a wave's arrays, PER numLoops slots per job; slot is the sample's first.  false when the
// thread has no sample.
template <int T, int PER, int D>
__device__ __forceinline__ bool vp_hyp_sample(int numLoops, double *slots, unsigned int *counts, int &j, int &smp,
                                              double *&slot)
{
  const int per = (numLoops + T - 1) / T;
  j = blockIdx.x / per;
  smp = (blockIdx.x - j * per) * T + threadIdx.x;
  if (smp >= numLoops) return false;
  const size_t first = (size_t)j * PER * numLoops + (size_t)PER * smp;
  slot = slots + first * D;
  for (int r = 0; r < PER; r++) { slot[D * r] = CUDART_NAN; counts[first + r] = 0; }
  return true;
}

// The K sums of a full warp's v, left in every lane: a fixed xor butterfly (a + b and b + a round alike, so every lane
// holds the same bits, and the order depends on nothing but the lanes' values).
template <int K>
__device__ __forceinline__ void vp_warp_sum(double (&v)[K])
{
#pragma unroll
  for (int o = 16; o; o >>= 1)
#pragma unroll
    for (int j = 0; j < K; j++) v[j] += __shfl_xor_sync(0xffffffffu, v[j], o);
}

// The largest key of a full warp, in every lane (a xor butterfly).
__device__ __forceinline__ unsigned long long vp_warp_max(unsigned long long key)
{
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const unsigned long long t = __shfl_xor_sync(0xffffffffu, key, o);
    key = t > key ? t : key;
  }
  return key;
}

// The packed arg-max of a warp's slots, all of one job: key = count << 32 | ~slot for a live slot (the most inliers,
// then the lowest slot), 0 otherwise; a butterfly, then lane 0's atomicMax of the key into *best and its addition of the
// warp's live slots to *numLive.  count is read for a live slot only.
__device__ __forceinline__ void vp_argmax_warp(bool live, const unsigned int *count, int slot, unsigned long long *best,
                                               unsigned long long *numLive)
{
  const unsigned long long key =
      vp_warp_max(live ? ((unsigned long long)*count << 32) | (unsigned int)~slot : 0ull);
  const unsigned int nl = __popc(__ballot_sync(0xffffffffu, live));
  if ((threadIdx.x & 31) == 0) {
    if (key) atomicMax(best, key);
    if (nl) atomicAdd(numLive, (unsigned long long)nl);
  }
}

// The Rodrigues rotation exp([w]x) = I + A [w]x + B [w]x^2, A = sin th / th, B = 2 sin^2(th / 2) / th^2 (A = 1, B = 1/2
// at th = 0): the update of absolute pose's refinement and of bundle adjustment.
__device__ __forceinline__ void vp_rodrigues(const double *w, double (&Q)[9])
{
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], th = sqrt(th2);
  double A = 1.0, B = 0.5;
  if (th2 != 0.0) {
    const double sh = sin(0.5 * th);
    A = sin(th) / th;
    B = 2.0 * sh * sh / th2;
  }
  const double W[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      const double W2 = W[3 * i] * W[j] + W[3 * i + 1] * W[3 + j] + W[3 * i + 2] * W[6 + j];
      Q[3 * i + j] = (i == j ? 1.0 : 0.0) + A * W[3 * i + j] + B * W2;
    }
}

// The left rotation update R1 = Q R with Q = exp([w]x) (vp_rodrigues), Q kept for the translation update, which
// differs between absolute pose and bundle adjustment.
__device__ __forceinline__ void vp_rotate(const double *w, const double *R, double *R1, double (&Q)[9])
{
  vp_rodrigues(w, Q);
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) R1[3 * i + j] = Q[3 * i] * R[j] + Q[3 * i + 1] * R[3 + j] + Q[3 * i + 2] * R[6 + j];
}

// Cholesky of the symmetric A (N x N, its lower triangle read); false when a pivot is not > 0 or not finite.  L is
// lower, packed row by row.
template <int N>
__device__ __forceinline__ bool vp_chol(const double (&A)[N][N], double *L)
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

// x = A^-1 b from the packed factor of vp_chol (forward, then backward substitution)
template <int N>
__device__ __forceinline__ void vp_chol_solve(const double *L, const double (&b)[N], double (&x)[N])
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

// The Levenberg-Marquardt damping lambda clamp(d, 1e-6, 1e32) added to a diagonal entry d of bundle adjustment and
// global positioning (to the scale block and the point and camera diagonals there, each by its own d).
__device__ __forceinline__ double vp_damping(double d, double lam) { return lam * fmin(fmax(d, 1e-6), 1e32); }

// The robust losses of cs_bundle_adjust_intrinsics and cs_global_positioning (1 soft-L1, 2 Cauchy) at s of scale c2:
// c^2 rho(s / c^2), and *w2 = rho'(s / c^2) when w2 is given.
__device__ __forceinline__ double vp_loss(int loss, double c2, double s, double *w2)
{
  const double u = s / c2;
  if (loss == 1) {
    const double q = sqrt(1.0 + u);
    if (w2) *w2 = 1.0 / q;
    return c2 * (2.0 * u / (q + 1.0));
  }
  if (w2) *w2 = 1.0 / (1.0 + u);
  return c2 * log1p(u);
}

// A valid member (a, f) of a track, the rule of triangulation and bundle adjustment: a known image, a feature inside
// its set, a finite position (x, y).  Cam is the call's camera table entry, with the set's pts and n.
template <class Cam>
__device__ __forceinline__ bool tr_member(const Cam *cams, int numImages, int2 af, float &x, float &y)
{
  if ((unsigned)af.x >= (unsigned)numImages) return false;
  const Cam &c = cams[af.x];
  if ((unsigned)af.y >= (unsigned)c.n) return false;
  x = c.pts[af.y].xpos;
  y = c.pts[af.y].ypos;
  return isfinite(x) && isfinite(y);
}

// The reprojection inlier rule of triangulation and absolute pose.  u = P (X, 1) with P = K [R | t] row-major 3 x 4:
// the homogeneous pixel, u[2] the depth.  The explicit fma chain pins the arithmetic, so scoring, refits and the
// per-feature outputs see the same bits.
__device__ __forceinline__ void tr_project(const double *P, const double (&X)[3], double (&u)[3])
{
#pragma unroll
  for (int i = 0; i < 3; i++) u[i] = fma(P[4 * i], X[0], fma(P[4 * i + 1], X[1], fma(P[4 * i + 2], X[2], P[4 * i + 3])));
}

// The squared pixel error times the squared depth: (u0 - x u2)^2 + (u1 - y u2)^2.
__device__ __forceinline__ double tr_err2z2(const double (&u)[3], float x, float y)
{
  const double dx = fma(-(double)x, u[2], u[0]), dy = fma(-(double)y, u[2], u[1]);
  return fma(dx, dx, dy * dy);
}

// An inlier: depth > 0 and the squared pixel error strictly below maxError^2 (multiplied through by depth^2).
__device__ __forceinline__ bool tr_inlier(const double *P, const double (&X)[3], float x, float y, double thr2)
{
  double u[3];
  tr_project(P, X, u);
  return u[2] > 0.0 && tr_err2z2(u, x, y) < thr2 * (u[2] * u[2]);
}

// The per-observation output of triangulation, absolute pose and bundle adjustment: the inlier byte of tr_inlier's
// rule and the pixel error (inf behind the camera).
__device__ __forceinline__ void tr_reproject(const double *P, const double (&X)[3], float x, float y, double thr2,
                                             float &err, unsigned char &in)
{
  double u[3];
  tr_project(P, X, u);
  const double e2z2 = tr_err2z2(u, x, y);
  in = u[2] > 0.0 && e2z2 < thr2 * (u[2] * u[2]);
  err = u[2] > 0.0 ? (float)sqrt(e2z2 / (u[2] * u[2])) : CUDART_INF_F;
}

}  // namespace cs
