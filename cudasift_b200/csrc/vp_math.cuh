// vp_math.cuh -- the FP64 helpers that geometric verification (verify.cu) and triangulation (triangulate.cu) share:
// the counter-based sampler, the cyclic Jacobi eigen-decomposition and the calibrated coordinates of a pinhole K.
// tests/verify_oracle.py and tests/triangulate_oracle.py restate them in float64.
#pragma once

#include <cmath>

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

}  // namespace cs
