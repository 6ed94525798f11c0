// verify.cu -- geometric verification of a correspondence list: RANSAC for a fundamental matrix (7-point minimal solver)
// or a homography (4-point), sampled on the device with a counter-based generator, scored in FP32 on normalised
// coordinates, refitted once.  The rules (validity, sampler, residuals, output order) are stated in cudasift_b200.h at
// cs_verify_pairs; tests/verify_oracle.py restates them in float64.
//
// Eight launches, one host synchronisation (by the caller, after the result copy).  The valid pairs and the inliers are
// ordered lists of ordered_list.cuh: flags and compact build the first, refit's final mask and write the second.
//   1. flags     one thread per pair: valid (indices in range, four finite coordinates).
//   2. compact   the valid pairs' pixel coordinates (float4 x1 y1 x2 y2) and their input index, in input order, and the
//                valid count.
//   3. norm      one CTA: centroids c1, c2 and the common Hartley scale s in double, fixed-order reductions; writes the
//                normalised FP32 coordinates and resets the arg-max key and the counters.
//   4. hyp       one thread per sample: draws, the minimal solver in FP64, up to 3 models (slot sample*3 + root) stored
//                unit-norm in normalised coordinates; an empty slot holds NaN.  Zeroes its slots' inlier counts.
//   5. score     grid (model blocks, point chunks): point tiles in shared memory, one model per thread, integer counts.
//   6. argmax    packed atomicMax of (count << 32 | ~slot): the highest count, then the lowest slot.
//   7. refit     one CTA: the normal matrix of the best model's inliers (fixed-order double reduction), Jacobi, rank 2 for
//                F, re-score, keep the refit unless it has fewer inliers; the final mask (ballot words, CTA counts), the
//                pixel model and the statistics.
//   8. write     the input pairs {i, j} of the inliers, in input order.
//
// Every launch verifies a wave of jobs (cs_verify_pairs_batch; a single call is a wave of one job).  A device table
// (VerifyJob) gives each job its records, pairs, seed, inlier buffer and intrinsics, and the first CTA of its range in
// the row kernels (1, 2, 8: one CTA per LIST_ROWS pairs, each job on CTAs of its own) and among the point chunks of the
// scoring kernel (grid y: the model blocks).  A CTA finds its job by binary search over those bases, built on the host.
// Norm and refit run one CTA per job, hyp and argmax a fixed number of CTAs per job.  Per job, every kernel does what
// it does for a single call, in the same CTA shapes and reduction orders, so a job's results do not depend on the
// other jobs of its wave.
#include <algorithm>
#include <cmath>
#include <vector>
#include <math_constants.h>

#include "common.cuh"
#include "ordered_list.cuh"
#include "vp_math.cuh"

namespace cs {

#define VP_HYP_T 128          // samples per CTA of the hypothesis kernel
#define VP_SC_T 128           // models per CTA of the scoring kernel
#define VP_TILE 1024          // points per shared-memory tile
#define VP_CHUNK 1024         // points per scoring CTA (one tile: more CTAs than models alone would give)
#define VP_REFIT_T 256
#define VP_EPS 1e-9           // smallest pivot / collinearity cross product, normalised coordinates (entries of order 1)

struct VerifyState {
  double c1x, c1y, c2x, c2y, s;   // normalisation: u = s * (x - c)
  double model[9];                // the returned model, pixel coordinates
  unsigned long long best;        // packed arg-max key; 0 = no model
  unsigned long long samples, models;
  long long stats[8];
  float thr2;                     // (s * thresh)^2
  int numValid;
  int total;                      // final inlier count
  // cs_verify_essential: model holds E; the chosen pose; [0] its points in front, [1] the runner-up candidate's count
  double R[9], t[3];
  long long pose[2];
};

// One job of a wave, as the kernels read it.  Its pair scratch (masks, CTA counts, coordinates, input indices) starts
// at CTA rowBase of the wave's row space, its model slots at job * slots per job.
struct VerifyJob {
  const SiftPoint *s1, *s2;
  const int2 *pairs;
  int2 *inliers;
  unsigned long long seed;
  int n1, n2, numPairs, maxInliers;
  int rowBase;                    // its first CTA of the flags / compact / write kernels
  int scoreBase;                  // its first CTA of the scoring kernel
  VerifyCalib cal;                // read by the essential kernels only
};

// ---- shared helpers (host and device); vp_splitmix64, vp_jacobi, vp_calibrate and vp_draw are in vp_math.cuh --------
__host__ __device__ inline void vp_mul33(const double *a, const double *b, double *c)
{
  for (int r = 0; r < 3; r++)
    for (int k = 0; k < 3; k++) c[3 * r + k] = a[3 * r] * b[k] + a[3 * r + 1] * b[3 + k] + a[3 * r + 2] * b[6 + k];
}

// F's output scaling: unit Frobenius norm, the largest-magnitude entry (the first of equals) positive; false for zero
__host__ __device__ inline bool vp_unit_sign(double *m)
{
  double n = 0.0;
  int big = 0;
  for (int k = 0; k < 9; k++) {
    n += m[k] * m[k];
    if (fabs(m[k]) > fabs(m[big])) big = k;
  }
  if (!(n > 0.0) || !isfinite(n)) return false;
  const double f = (m[big] < 0 ? -1.0 : 1.0) / sqrt(n);
  for (int k = 0; k < 9; k++) m[k] *= f;
  return true;
}

// a normalised-coordinate model to pixel coordinates and its output scale: H = T2^-1 Hn T1 with H[8] = 1,
// F = T2^T Fn T1 with F's output scaling (vp_unit_sign)
__host__ __device__ inline void vp_denormalise(const double *m, int model, double c1x, double c1y, double c2x, double c2y,
                                               double s, double *out)
{
  const double T1[9] = {s, 0, -s * c1x, 0, s, -s * c1y, 0, 0, 1};
  double L[9], t[9];
  if (model == CS_GEOM_HOMOGRAPHY) {
    const double T2i[9] = {1.0 / s, 0, c2x, 0, 1.0 / s, c2y, 0, 0, 1};
    for (int k = 0; k < 9; k++) L[k] = T2i[k];
  } else {
    const double T2t[9] = {s, 0, 0, 0, s, 0, -s * c2x, -s * c2y, 1};
    for (int k = 0; k < 9; k++) L[k] = T2t[k];
  }
  vp_mul33(L, m, t);
  vp_mul33(t, T1, out);
  if (model == CS_GEOM_HOMOGRAPHY) {
    const double d = out[8];
    if (d != 0.0) for (int k = 0; k < 9; k++) out[k] /= d;
  } else {
    vp_unit_sign(out);
  }
}

// ---- device routines ----------------------------------------------------------------------------------------------
// Null space of an M x 9 system (M = 5, 7 or 8): Gaussian elimination with partial pivoting on columns 0..M-1, then back
// substitution for each free column f = M..8 (x_f = 1, the other free entries 0).  false when a pivot is below VP_EPS.
template <int M>
__host__ __device__ bool vp_nullspace(double (&A)[M][9], double (&N)[9 - M][9])
{
#pragma unroll
  for (int c = 0; c < M; c++) {
    int p = c;
    double best = fabs(A[c][c]);
#pragma unroll
    for (int r = c + 1; r < M; r++)
      if (fabs(A[r][c]) > best) { best = fabs(A[r][c]); p = r; }
    if (!(best >= VP_EPS)) return false;
#pragma unroll
    for (int r = c + 1; r < M; r++)
      if (r == p) {
#pragma unroll
        for (int j = 0; j < 9; j++) { const double t = A[c][j]; A[c][j] = A[r][j]; A[r][j] = t; }
      }
#pragma unroll
    for (int r = c + 1; r < M; r++) {
      const double f = A[r][c] / A[c][c];
#pragma unroll
      for (int j = c; j < 9; j++) A[r][j] -= f * A[c][j];
    }
  }
#pragma unroll
  for (int f = M; f < 9; f++) {
    double *x = N[f - M];
#pragma unroll
    for (int j = M; j < 9; j++) x[j] = j == f ? 1.0 : 0.0;
#pragma unroll
    for (int r = M - 1; r >= 0; r--) {
      double acc = 0.0;
#pragma unroll
      for (int j = r + 1; j < 9; j++) acc += A[r][j] * x[j];
      x[r] = -acc / A[r][r];
    }
  }
  return true;
}

__device__ inline double vp_det3(const double *m)
{
  return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}

// Real roots of c0 + c1 a + c2 a^2 + c3 a^3 (closed form, unpolished, unordered).  A coefficient below 1e-10 of the
// largest counts as zero from the top (cubic -> quadratic -> linear).
__device__ int vp_cubic_roots(const double *c, double *roots)
{
  double cm = 0.0;
  for (int k = 0; k < 4; k++) cm = fmax(cm, fabs(c[k]));
  if (!(cm > 0.0)) return 0;
  int n = 0;
  if (fabs(c[3]) > 1e-10 * cm) {
    const double a = c[2] / c[3], b = c[1] / c[3], d = c[0] / c[3];
    const double p = b - a * a / 3.0, q = 2.0 * a * a * a / 27.0 - a * b / 3.0 + d;
    const double disc = 0.25 * q * q + p * p * p / 27.0;
    if (disc > 0.0) {
      const double sq = sqrt(disc);
      roots[n++] = cbrt(-0.5 * q + sq) + cbrt(-0.5 * q - sq) - a / 3.0;
    } else if (p == 0.0) {
      roots[n++] = -a / 3.0;
    } else {
      const double r = sqrt(-p / 3.0);
      const double arg = fmin(1.0, fmax(-1.0, 1.5 * q / p * sqrt(-3.0 / p)));
      const double phi = acos(arg);
      for (int k = 0; k < 3; k++) roots[n++] = 2.0 * r * cos(phi / 3.0 - 2.0 * M_PI * k / 3.0) - a / 3.0;
    }
  } else if (fabs(c[2]) > 1e-10 * cm) {
    const double disc = c[1] * c[1] - 4.0 * c[2] * c[0];
    if (disc >= 0.0) {
      const double qq = -0.5 * (c[1] + (c[1] >= 0 ? 1.0 : -1.0) * sqrt(disc));
      roots[n++] = qq / c[2];
      if (qq != 0.0) roots[n++] = c[0] / qq;
    }
  } else if (fabs(c[1]) > 1e-10 * cm) {
    roots[n++] = -c[0] / c[1];
  }
  return n;
}

__device__ inline bool vp_store_unit(double *slot, const double *m)
{
  double n = 0.0;
  for (int k = 0; k < 9; k++) n += m[k] * m[k];
  if (!(n > 0.0) || !isfinite(n)) return false;
  const double f = 1.0 / sqrt(n);
  for (int k = 0; k < 9; k++) slot[k] = m[k] * f;
  return true;
}

// FP32 inlier tests on normalised coordinates p = {u1, v1, u2, v2}, against thr2 = (s * thresh)^2.  The explicit fmaf
// chain pins the arithmetic: scoring, the refit's counts and the final mask see the same bits.
__device__ __forceinline__ bool vp_inlier(const float *m, float4 p, float thr2, bool homography)
{
  if (homography) {                    // |(X, Y) / w - x2|^2 < thr2, multiplied through by w^2 (no division)
    const float w = fmaf(m[6], p.x, fmaf(m[7], p.y, m[8]));
    const float X = fmaf(m[0], p.x, fmaf(m[1], p.y, m[2]));
    const float Y = fmaf(m[3], p.x, fmaf(m[4], p.y, m[5]));
    const float dx = fmaf(-p.z, w, X), dy = fmaf(-p.w, w, Y);
    return fmaf(dx, dx, dy * dy) < thr2 * (w * w);
  }
  const float a0 = fmaf(m[0], p.x, fmaf(m[1], p.y, m[2]));
  const float a1 = fmaf(m[3], p.x, fmaf(m[4], p.y, m[5]));
  const float a2 = fmaf(m[6], p.x, fmaf(m[7], p.y, m[8]));
  const float b0 = fmaf(m[0], p.z, fmaf(m[3], p.w, m[6]));
  const float b1 = fmaf(m[1], p.z, fmaf(m[4], p.w, m[7]));
  const float num = fmaf(p.z, a0, fmaf(p.w, a1, a2));
  const float den = fmaf(a0, a0, fmaf(a1, a1, fmaf(b0, b0, b1 * b1)));
  return num * num < thr2 * den;
}

// ---- kernels ----------------------------------------------------------------------------------------------------------
// The scratch of a wave: per row CTA LIST_ROWS / 32 mask words, one count and LIST_ROWS coordinates and input indices;
// per job `slots` model slots, their counts and one state.
struct VerifyWave {
  const VerifyJob *jobs;
  int numJobs, slots;
  unsigned int *masks, *counts;
  float4 *xy, *un;
  int *orig;
  double *models;
  unsigned int *slotCounts;
  VerifyState *st;
};

// One job's part of a wave's scratch.
struct VerifyJobScratch {
  unsigned int *masks, *counts;
  float4 *xy, *un;
  int *orig;
  double *models;
  unsigned int *slotCounts;
  VerifyState *st;
};

__device__ __forceinline__ VerifyJobScratch vp_job_scratch(const VerifyWave &w, int j)
{
  const size_t r = (size_t)w.jobs[j].rowBase;
  return {w.masks + r * (LIST_ROWS / 32), w.counts + r, w.xy + r * LIST_ROWS, w.un + r * LIST_ROWS,
          w.orig + r * LIST_ROWS, w.models + (size_t)j * w.slots * 9, w.slotCounts + (size_t)j * w.slots, w.st + j};
}

__global__ void __launch_bounds__(LIST_ROWS)
vp_flags_kernel(VerifyWave w)
{
  const int j = table_find(w.jobs, w.numJobs, &VerifyJob::rowBase, (int)blockIdx.x);
  const VerifyJob &job = w.jobs[j];
  const VerifyJobScratch js = vp_job_scratch(w, j);
  const SiftPoint *__restrict__ s1 = job.s1, *__restrict__ s2 = job.s2;
  const int n1 = job.n1, n2 = job.n2, numPairs = job.numPairs;
  const int b = blockIdx.x - job.rowBase;
  const int k = b * LIST_ROWS + threadIdx.x;
  bool keep = false;
  if (k < numPairs) {
    const int2 p = job.pairs[k];
    if (p.x >= 0 && p.x < n1 && p.y >= 0 && p.y < n2)
      keep = isfinite(s1[p.x].xpos) && isfinite(s1[p.x].ypos) && isfinite(s2[p.y].xpos) && isfinite(s2[p.y].ypos);
  }
  list_flag(keep, k, numPairs, js.masks, js.counts, b);
}

__global__ void __launch_bounds__(LIST_ROWS)
vp_compact_kernel(VerifyWave w)
{
  const int j = table_find(w.jobs, w.numJobs, &VerifyJob::rowBase, (int)blockIdx.x);
  const VerifyJob &job = w.jobs[j];
  const VerifyJobScratch js = vp_job_scratch(w, j);
  const int b = blockIdx.x - job.rowBase;
  bool bit;
  const unsigned int pos = list_position(js.masks, js.counts, job.numPairs, b, &bit,
                                         reinterpret_cast<unsigned int *>(&js.st->numValid));
  if (bit) {
    const int k = b * LIST_ROWS + threadIdx.x;
    const int2 p = job.pairs[k];
    js.xy[pos] = make_float4(job.s1[p.x].xpos, job.s1[p.x].ypos, job.s2[p.y].xpos, job.s2[p.y].ypos);
    js.orig[pos] = k;
  }
}

// block-wide sum of 4 doubles in a fixed order (xor butterfly per warp, then warp 0 over the warp partials)
__device__ void vp_block_sum4(double (&v)[4], double (*s_red)[4])
{
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < 4; j++)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[j] += __shfl_xor_sync(0xffffffffu, v[j], o);
  if (lane == 0)
    for (int j = 0; j < 4; j++) s_red[w][j] = v[j];
  __syncthreads();
  if (w == 0) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
      double t = lane < (int)(blockDim.x >> 5) ? s_red[lane][j] : 0.0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if (lane == 0) s_red[0][j] = t;
    }
  }
  __syncthreads();
  for (int j = 0; j < 4; j++) v[j] = s_red[0][j];
  __syncthreads();
}

// one CTA per job
__global__ void __launch_bounds__(1024)
vp_norm_kernel(VerifyWave w, float thresh)
{
  __shared__ double s_red[32][4];
  const VerifyJobScratch js = vp_job_scratch(w, blockIdx.x);
  const float4 *__restrict__ xy = js.xy;
  float4 *__restrict__ un = js.un;
  VerifyState *st = js.st;
  const int n = st->numValid;
  double v[4] = {0, 0, 0, 0};
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const float4 p = xy[k];
    v[0] += p.x; v[1] += p.y; v[2] += p.z; v[3] += p.w;
  }
  vp_block_sum4(v, s_red);
  const double c1x = n ? v[0] / n : 0.0, c1y = n ? v[1] / n : 0.0, c2x = n ? v[2] / n : 0.0, c2y = n ? v[3] / n : 0.0;
  double d[4] = {0, 0, 0, 0};
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const float4 p = xy[k];
    d[0] += sqrt((p.x - c1x) * (p.x - c1x) + (p.y - c1y) * (p.y - c1y));
    d[1] += sqrt((p.z - c2x) * (p.z - c2x) + (p.w - c2y) * (p.w - c2y));
  }
  vp_block_sum4(d, s_red);
  const double mean = n ? (d[0] + d[1]) / (2.0 * n) : 0.0;
  const double s = mean > 0.0 ? sqrt(2.0) / mean : 0.0;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const float4 p = xy[k];
    un[k] = make_float4((float)((p.x - c1x) * s), (float)((p.y - c1y) * s), (float)((p.z - c2x) * s),
                        (float)((p.w - c2y) * s));
  }
  if (threadIdx.x == 0) {
    st->c1x = c1x; st->c1y = c1y; st->c2x = c2x; st->c2y = c2y; st->s = s;
    const double t = s * (double)thresh;
    st->thr2 = (float)(t * t);
    st->best = 0; st->samples = 0; st->models = 0;
  }
}

__device__ inline double vp_cross(double ax, double ay, double bx, double by, double cx, double cy)
{
  return (bx - ax) * (cy - ay) - (by - ay) * (cx - ax);
}

// One thread's sample in a hypothesis kernel: its job, that job's scratch, the sample's first slot and index.
struct VerifySample {
  const VerifyJob *job;
  VerifyJobScratch js;
  double *slot;
  int smp;
};

// The prologue of the hypothesis kernels: vp_hyp_sample (PER slots of 9 doubles per sample), then the scale check and
// the K draws of the sample into idx.  false when the thread has no sample or the sample has no draw.
template <int PER, int K>
__device__ __forceinline__ bool vp_hyp_prologue(const VerifyWave &w, int numLoops, VerifySample &h, int (&idx)[K])
{
  int j;
  if (!vp_hyp_sample<VP_HYP_T, PER, 9>(numLoops, w.models, w.slotCounts, j, h.smp, h.slot)) return false;
  h.job = w.jobs + j;
  h.js = vp_job_scratch(w, j);
  return h.js.st->s > 0.0 && vp_draw<K>(h.job->seed, h.smp, h.js.st->numValid, idx);
}

__global__ void __launch_bounds__(VP_HYP_T)
vp_hyp_kernel(VerifyWave w, int numLoops, int model)
{
  VerifySample h;
  if (model == CS_GEOM_HOMOGRAPHY) {
    int idx[4];
    if (!vp_hyp_prologue<3>(w, numLoops, h, idx)) return;
    const float4 *__restrict__ xy = h.js.xy;
    const VerifyState *st = h.js.st;
    const double s = st->s, c1x = st->c1x, c1y = st->c1y, c2x = st->c2x, c2y = st->c2y;
    double u[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const float4 p = xy[idx[i]];
      u[i][0] = (p.x - c1x) * s; u[i][1] = (p.y - c1y) * s; u[i][2] = (p.z - c2x) * s; u[i][3] = (p.w - c2y) * s;
    }
    const int tri[4][3] = {{0, 1, 2}, {0, 1, 3}, {0, 2, 3}, {1, 2, 3}};
#pragma unroll
    for (int t = 0; t < 4; t++)
#pragma unroll
      for (int im = 0; im < 2; im++) {
        const double *a = u[tri[t][0]] + 2 * im, *b = u[tri[t][1]] + 2 * im, *c = u[tri[t][2]] + 2 * im;
        if (!(fabs(vp_cross(a[0], a[1], b[0], b[1], c[0], c[1])) >= VP_EPS)) return;
      }
    double A[8][9], N[1][9];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const double x = u[i][0], y = u[i][1], X = u[i][2], Y = u[i][3];
      const double r1[9] = {x, y, 1, 0, 0, 0, -X * x, -X * y, -X}, r2[9] = {0, 0, 0, x, y, 1, -Y * x, -Y * y, -Y};
#pragma unroll
      for (int j = 0; j < 9; j++) { A[2 * i][j] = r1[j]; A[2 * i + 1][j] = r2[j]; }
    }
    if (!vp_nullspace<8>(A, N)) return;
    vp_store_unit(h.slot, N[0]);
    return;
  }
  int idx[7];
  if (!vp_hyp_prologue<3>(w, numLoops, h, idx)) return;
  const float4 *__restrict__ xy = h.js.xy;
  const VerifyState *st = h.js.st;
  const double s = st->s, c1x = st->c1x, c1y = st->c1y, c2x = st->c2x, c2y = st->c2y;
  double A[7][9], N[2][9];
#pragma unroll
  for (int i = 0; i < 7; i++) {
    const float4 p = xy[idx[i]];
    const double x = (p.x - c1x) * s, y = (p.y - c1y) * s, X = (p.z - c2x) * s, Y = (p.w - c2y) * s;
    const double r[9] = {X * x, X * y, X, Y * x, Y * y, Y, x, y, 1};
#pragma unroll
    for (int j = 0; j < 9; j++) A[i][j] = r[j];
  }
  if (!vp_nullspace<7>(A, N)) return;
  // det(a F1 + (1 - a) F2) = det(F2 + a (F1 - F2)) = c0 + c1 a + c2 a^2 + c3 a^3, from its values at a = 0, 1, -1, 2
  double D[9], M[9], p[4];
  for (int k = 0; k < 9; k++) D[k] = N[0][k] - N[1][k];
  const double at[4] = {0.0, 1.0, -1.0, 2.0};
  for (int q = 0; q < 4; q++) {
    for (int k = 0; k < 9; k++) M[k] = N[1][k] + at[q] * D[k];
    p[q] = vp_det3(M);
  }
  double c[4];
  c[0] = p[0];
  c[2] = 0.5 * (p[1] + p[2]) - p[0];
  const double a = 0.5 * (p[1] - p[2]), b = p[3] - p[0] - 4.0 * c[2];
  c[3] = (b - 2.0 * a) / 6.0;
  c[1] = a - c[3];
  // two Newton steps per root on the determinant itself (the interpolated cubic's derivative as the slope), then
  // ascending order
  double roots[3];
  const int nr = vp_cubic_roots(c, roots);
  for (int k = 0; k < nr; k++)
    for (int it = 0; it < 2; it++) {
      const double x = roots[k];
      const double d = (3.0 * c[3] * x + 2.0 * c[2]) * x + c[1];
      if (d == 0.0) break;
      for (int j = 0; j < 9; j++) M[j] = N[1][j] + x * D[j];
      const double y = x - vp_det3(M) / d;
      if (isfinite(y)) roots[k] = y;
    }
  for (int i = 1; i < nr; i++)
    for (int j = i; j > 0 && roots[j] < roots[j - 1]; j--) { const double t = roots[j]; roots[j] = roots[j - 1]; roots[j - 1] = t; }
  int r = 0;
  for (int k = 0; k < nr; k++) {
    for (int j = 0; j < 9; j++) M[j] = roots[k] * N[0][j] + (1.0 - roots[k]) * N[1][j];
    if (vp_store_unit(h.slot + 9 * r, M)) r++;
  }
}

// one thread per slot (F) or per sample's slot 3s (H: its only model), VP_CHUNK points per CTA; grid (point chunks of
// all jobs, model blocks): a job's chunks are the idivup(numPairs, VP_CHUNK) CTAs from its scoreBase on
__global__ void __launch_bounds__(VP_SC_T)
vp_score_kernel(VerifyWave w, int model)
{
  __shared__ float4 s_p[VP_TILE];
  const int j = table_find(w.jobs, w.numJobs, &VerifyJob::scoreBase, (int)blockIdx.x);
  const VerifyJobScratch js = vp_job_scratch(w, j);
  const float4 *__restrict__ un = js.un;
  const double *__restrict__ models = js.models;
  const int numSlots = w.slots;
  const int n = js.st->numValid;
  const int p0 = (blockIdx.x - w.jobs[j].scoreBase) * VP_CHUNK;
  if (p0 >= n) return;
  const int p1 = min(n, p0 + VP_CHUNK);
  const int slot = (blockIdx.y * VP_SC_T + threadIdx.x) * (model == CS_GEOM_HOMOGRAPHY ? 3 : 1);
  float m[9];
  bool live = slot < numSlots && !isnan(models[(size_t)slot * 9]);
  if (live)
    for (int k = 0; k < 9; k++) m[k] = (float)models[(size_t)slot * 9 + k];
  const float thr2 = js.st->thr2;
  const bool homography = model == CS_GEOM_HOMOGRAPHY;
  unsigned int cnt = 0;
  for (int t0 = p0; t0 < p1; t0 += VP_TILE) {
    const int tn = min(VP_TILE, p1 - t0);
    __syncthreads();
    for (int k = threadIdx.x; k < tn; k += VP_SC_T) s_p[k] = un[t0 + k];
    __syncthreads();
    if (live)
      for (int k = 0; k < tn; k++) cnt += vp_inlier(m, s_p[k], thr2, homography);
  }
  if (live && cnt) atomicAdd(&js.slotCounts[slot], cnt);
}

// perSample: slots per sample (3 for F and H, 10 for E); a sample counts when its first slot is live.
// idivup(slots, 256) CTAs per job, so that no warp holds two jobs' slots.
__global__ void __launch_bounds__(256)
vp_argmax_kernel(VerifyWave w, int perSample)
{
  const int numSlots = w.slots, per = (numSlots + 255) / 256, j = blockIdx.x / per;
  const VerifyJobScratch js = vp_job_scratch(w, j);
  const double *__restrict__ models = js.models;
  const unsigned int *__restrict__ counts = js.slotCounts;
  VerifyState *st = js.st;
  const int slot = (blockIdx.x - j * per) * 256 + threadIdx.x;
  const bool live = slot < numSlots && !isnan(models[(size_t)slot * 9]);
  vp_argmax_warp(live, counts + slot, slot, &st->best, &st->models);
  const unsigned int ns = __popc(__ballot_sync(0xffffffffu, live && slot % perSample == 0));
  if ((threadIdx.x & 31) == 0 && ns) atomicAdd(&st->samples, (unsigned long long)ns);
}

// block-wide sum of an int (fixed order; the result in every thread)
__device__ int vp_block_count(int v, int *s_cnt)
{
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane == 0) s_cnt[w] = v;
  __syncthreads();
  int t = 0;
  for (int k = 0; k < VP_REFIT_T / 32; k++) t += s_cnt[k];
  return t;
}

// The final mask of a refit CTA, in the layout of an ordered list (ordered_list.cuh): ballot words per 32 points of the
// FP32 test with m (all clear when m is null), then counts per LIST_ROWS points; returns the total in every thread.
__device__ int vp_final_mask(const float *m, const float4 *__restrict__ un, int n, float thr2, bool homography,
                             unsigned int *__restrict__ masks, unsigned int *__restrict__ blockCounts, int *s_cnt)
{
  const int lane = threadIdx.x & 31;
  if (m) {
    for (int k0 = 0; k0 < n; k0 += VP_REFIT_T) {
      const int k = k0 + threadIdx.x;
      const bool in = k < n && vp_inlier(m, un[k], thr2, homography);
      const unsigned int bal = __ballot_sync(0xffffffffu, in);
      if (lane == 0 && k < n) masks[k >> 5] = bal;
    }
  } else {
    for (int k = threadIdx.x; k < list_words(n); k += VP_REFIT_T) masks[k] = 0u;
  }
  __syncthreads();
  const int words = list_words(n);
  int tot = 0;
  for (int b = threadIdx.x; b < list_ctas(n); b += VP_REFIT_T) {
    unsigned int t = 0;
    for (int q = b * (LIST_ROWS / 32); q < min(words, (b + 1) * (LIST_ROWS / 32)); q++) t += __popc(masks[q]);
    blockCounts[b] = t;
    tot += (int)t;
  }
  return vp_block_count(tot, s_cnt);
}

// The 45 upper-triangle entries of one thread's normal-matrix partial sums, summed over each warp into s_nm[warp].
__device__ __forceinline__ void vp_warp_normal(const double (&acc)[45], double (*s_nm)[45])
{
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int e = 0; e < 45; e++) {
    double v = acc[e];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) s_nm[w][e] = v;
  }
}

// The symmetric 9x9 normal matrix from the warps' sums (in warp order), and its smallest eigenvector (Jacobi).
__device__ void vp_smallest_eigvec(const double (*s_nm)[45], double (&f)[9])
{
  double A[9][9], V[9][9];
  int e = 0;
  for (int i = 0; i < 9; i++)
    for (int j = i; j < 9; j++) {
      double t = 0.0;
      for (int q = 0; q < VP_REFIT_T / 32; q++) t += s_nm[q][e];
      A[i][j] = A[j][i] = t;
      e++;
    }
  vp_jacobi<9>(A, V);
  int lo = 0;
  for (int i = 1; i < 9; i++) if (A[i][i] < A[lo][lo]) lo = i;
  for (int i = 0; i < 9; i++) f[i] = V[i][lo];
}

__global__ void __launch_bounds__(LIST_ROWS)
vp_write_kernel(VerifyWave w)
{
  const int j = table_find(w.jobs, w.numJobs, &VerifyJob::rowBase, (int)blockIdx.x);
  const VerifyJob &job = w.jobs[j];
  const VerifyJobScratch js = vp_job_scratch(w, j);
  const int b = blockIdx.x - job.rowBase;
  const int n = js.st->numValid;
  if (b * LIST_ROWS >= n) return;                   // the whole CTA: no thread reaches the scan's barriers
  bool bit;
  const unsigned int pos = list_position(js.masks, js.counts, n, b, &bit, nullptr);
  if (bit && pos < (unsigned int)job.maxInliers) job.inliers[pos] = job.pairs[js.orig[b * LIST_ROWS + threadIdx.x]];
}

// ---- the calibrated path (cs_verify_essential) -------------------------------------------------------------------------
// Steps 1-3 and 5, 6, 8 are the kernels above (scoring with the F test on Fn = T2^-T K2^-T E K1^-1 T1^-1); step 4 is
// vp_hyp5_kernel (10 slots per sample) and step 7 vp_refit_kernel<true>.  The rules are stated in
// cudasift_b200.h at cs_verify_essential.
#define VP_E_SLOTS 10            // models per sample of the 5-point solver
#define VP_E_PIVOT 1e-12         // Gauss-Jordan pivot, relative to the largest |entry| of the 10x20 matrix
#define VP_E_LEAD 1e-12          // leading coefficients of the degree-10 polynomial at or below this (relative) are dropped
#define VP_E_REM 1e-14           // a Sturm remainder at or below this (relative to its dividend) ends the sequence
#define VP_E_WIDTH 1e-10         // root refinement: bisection down to this width (relative to max(1, |end|))
#define VP_E_STACK 64            // isolation intervals pending at once
#define VP_E_PARALLEL 1e-12      // cheirality: rays whose sin^2(angle) is at or below this are not in front

// G = K^-1 T^-1: normalised coordinates -> calibrated, T the normalisation u = s (x - c)
__host__ __device__ inline void vp_norm_to_calib(const double *K, double cx, double cy, double s, double *G)
{
  const double Ki[9] = {1.0 / K[0], -K[1] / (K[0] * K[4]), (K[1] * K[5] - K[2] * K[4]) / (K[0] * K[4]),
                        0, 1.0 / K[4], -K[5] / K[4], 0, 0, 1};
  const double Ti[9] = {1.0 / s, 0, cx, 0, 1.0 / s, cy, 0, 0, 1};
  vp_mul33(Ki, Ti, G);
}

// TK = T K, the inverse of G
__host__ __device__ inline void vp_calib_to_norm(const double *K, double cx, double cy, double s, double *TK)
{
  const double T[9] = {s, 0, -s * cx, 0, s, -s * cy, 0, 0, 1};
  vp_mul33(T, K, TK);
}

// out = A^T M B: Fn = G2^T E G1, and back E = TK2^T Fn TK1
__host__ __device__ inline void vp_sandwich(const double *A, const double *M, const double *B, double *out)
{
  double At[9], t[9];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) At[3 * r + c] = A[3 * c + r];
  vp_mul33(At, M, t);
  vp_mul33(t, B, out);
}

// E = (T2 K2)^T Fn (T1 K1): the essential matrix of a stored Fn, under the job's normalisation v
__host__ __device__ inline void vp_fn_to_e(const VerifyCalib &cal, const VerifyState &v, const double *fn, double *E)
{
  double TK1[9], TK2[9];
  vp_calib_to_norm(cal.K1, v.c1x, v.c1y, v.s, TK1);
  vp_calib_to_norm(cal.K2, v.c2x, v.c2y, v.s, TK2);
  vp_sandwich(TK2, fn, TK1, E);
}

// Polynomials of degree <= 3 in (x, y, z): 20 coefficients in Nister's monomial order
//   x^3 y^3 x^2y xy^2 x^2z x^2 y^2z y^2 xyz xy | xz^2 xz x yz^2 yz y z^3 z^2 z 1
__host__ __device__ constexpr int vp_mono(int a, int b, int c)      // the slot of x^a y^b z^c
{
  return a == 3 ? 0 : b == 3 ? 1 : (a == 2 && b == 1) ? 2 : (a == 1 && b == 2) ? 3 : (a == 2 && c == 1) ? 4
       : a == 2 ? 5 : (b == 2 && c == 1) ? 6 : b == 2 ? 7 : (a == 1 && b == 1 && c == 1) ? 8 : (a == 1 && b == 1) ? 9
       : (a == 1 && c == 2) ? 10 : (a == 1 && c == 1) ? 11 : a == 1 ? 12 : (b == 1 && c == 2) ? 13
       : (b == 1 && c == 1) ? 14 : b == 1 ? 15 : c == 3 ? 16 : c == 2 ? 17 : c == 1 ? 18 : 19;
}
__host__ __device__ constexpr int vp_mono_exp(int k)                // the exponents of slot k, a << 4 | b << 2 | c
{
  return k == 0 ? 0x30 : k == 1 ? 0x0C : k == 2 ? 0x24 : k == 3 ? 0x18 : k == 4 ? 0x21 : k == 5 ? 0x20 : k == 6 ? 0x09
       : k == 7 ? 0x08 : k == 8 ? 0x15 : k == 9 ? 0x14 : k == 10 ? 0x12 : k == 11 ? 0x11 : k == 12 ? 0x10
       : k == 13 ? 0x06 : k == 14 ? 0x05 : k == 15 ? 0x04 : k == 16 ? 0x03 : k == 17 ? 0x02 : k == 18 ? 0x01 : 0x00;
}
__host__ __device__ constexpr int vp_mono_deg(int e) { return (e >> 4) + ((e >> 2) & 3) + (e & 3); }

// r += sign * p * q for p of degree <= DP and q of degree <= DQ, DP + DQ <= 3
template <int DP, int DQ>
__host__ __device__ __forceinline__ void vp_pmul(const double *p, const double *q, double sign, double *r)
{
#pragma unroll
  for (int i = 0; i < 20; i++) {
    if (vp_mono_deg(vp_mono_exp(i)) > DP) continue;
#pragma unroll
    for (int j = 0; j < 20; j++) {
      if (vp_mono_deg(vp_mono_exp(j)) > DQ) continue;
      const int a = vp_mono_exp(i), b = vp_mono_exp(j);
      r[vp_mono((a >> 4) + (b >> 4), ((a >> 2) & 3) + ((b >> 2) & 3), (a & 3) + (b & 3))] += sign * (p[i] * q[j]);
    }
  }
}

// out[0..na+nb] = a * b, coefficients in ascending powers
__host__ __device__ inline void vp_upoly_mul(const double *a, int na, const double *b, int nb, double *out)
{
  for (int k = 0; k <= na + nb; k++) out[k] = 0.0;
  for (int i = 0; i <= na; i++)
    for (int j = 0; j <= nb; j++) out[i + j] += a[i] * b[j];
}

__host__ __device__ inline double vp_horner(const double *c, int n, double x)
{
  double v = c[n];
  for (int k = n - 1; k >= 0; k--) v = v * x + c[k];
  return v;
}

// sign changes of the Sturm sequence at x (zeros skipped)
__host__ __device__ inline int vp_sturm_changes(const double (*S)[11], const int *deg, int ns, double x)
{
  int changes = 0;
  double prev = 0.0;
  for (int k = 0; k < ns; k++) {
    const double v = vp_horner(S[k], deg[k], x);
    if (v == 0.0) continue;
    if (prev != 0.0 && (v > 0.0) != (prev > 0.0)) changes++;
    prev = v;
  }
  return changes;
}

// The distinct real roots of c[0] + c[1] z + ... + c[n] z^n (n <= 10), ascending; returns their number.  Leading
// coefficients at or below VP_E_LEAD of the largest |c| are dropped.  Sturm sequence of the monic p: S0 = p,
// S1 = p' / n, S(k+1) = -rem(S(k-1), S(k)) scaled by 1 / |its leading coefficient|, ending when a remainder's largest
// |coefficient| is at or below VP_E_REM of its dividend's (leading remainder coefficients at or below VP_E_REM of that
// largest one are dropped).  Isolation: (-B, B], B = 1 + 2 max_k |a(n-k)|^(1/k) of the monic p (Fujiwara), bisected
// at midpoints, left half first, halves without a root dropped; an interval is refined as one root when it holds one
// root, is narrower than VP_E_WIDTH * max(1, |lo|, |hi|), or more than VP_E_STACK - 2 other intervals are pending
// (the stack then has no room for two halves).  Refinement: bisection to that width, on the sign of p
// when p changes sign across the interval, else on the Sturm count (the left half while it holds a root); then up to
// three Newton steps from the midpoint, each kept only while it stays inside the interval.
__host__ __device__ inline int vp_real_roots(const double *c, int n, double *roots)
{
  double cm = 0.0;
  for (int k = 0; k <= n; k++) cm = fmax(cm, fabs(c[k]));
  if (!(cm > 0.0) || !isfinite(cm)) return 0;
  while (n > 0 && !(fabs(c[n]) > VP_E_LEAD * cm)) n--;
  if (n == 0) return 0;
  double S[11][11];
  int deg[11];
  for (int k = 0; k <= n; k++) S[0][k] = c[k] / c[n];
  for (int k = 0; k < n; k++) S[1][k] = (k + 1) * S[0][k + 1] / n;
  deg[0] = n; deg[1] = n - 1;
  int ns = 2;
  while (deg[ns - 1] > 0) {
    const double *a = S[ns - 2], *b = S[ns - 1];
    const int da = deg[ns - 2], db = deg[ns - 1];
    double r[11], am = 0.0;
    for (int k = 0; k <= da; k++) { r[k] = a[k]; am = fmax(am, fabs(a[k])); }
    for (int k = da - db; k >= 0; k--) {
      const double q = r[db + k] / b[db];
      for (int j = 0; j <= db; j++) r[j + k] -= q * b[j];
    }
    double rm = 0.0;
    for (int k = 0; k < db; k++) rm = fmax(rm, fabs(r[k]));
    if (!(rm > VP_E_REM * am)) break;
    int dr = db - 1;
    while (dr > 0 && !(fabs(r[dr]) > VP_E_REM * rm)) dr--;
    const double f = -1.0 / fabs(r[dr]);
    for (int k = 0; k <= dr; k++) S[ns][k] = r[k] * f;
    deg[ns++] = dr;
  }
  double B = 0.0;                      // Fujiwara's bound 2 max |a(n-k)|^(1/k), plus 1
  for (int k = 1; k <= n; k++) B = fmax(B, pow(fabs(S[0][n - k]), 1.0 / k));
  B = 2.0 * B + 1.0;
  struct Iv { double lo, hi; int vlo, vhi; };
  Iv stack[VP_E_STACK];
  int top = 0, nr = 0;
  stack[top++] = {-B, B, vp_sturm_changes(S, deg, ns, -B), vp_sturm_changes(S, deg, ns, B)};
  while (top > 0 && nr < n) {
    Iv iv = stack[--top];
    const int cnt = iv.vlo - iv.vhi;
    if (cnt <= 0) continue;
    const double tol = VP_E_WIDTH * fmax(1.0, fmax(fabs(iv.lo), fabs(iv.hi)));
    if (cnt > 1 && iv.hi - iv.lo > tol && top + 2 <= VP_E_STACK) {
      const double mid = 0.5 * (iv.lo + iv.hi);
      const int vm = vp_sturm_changes(S, deg, ns, mid);
      if (vm > iv.vhi) stack[top++] = {mid, iv.hi, vm, iv.vhi};      // only halves that hold a root are kept
      if (iv.vlo > vm) stack[top++] = {iv.lo, mid, iv.vlo, vm};
      continue;
    }
    double lo = iv.lo, hi = iv.hi, plo = vp_horner(S[0], n, lo);
    int vlo = iv.vlo;
    const double phi = vp_horner(S[0], n, hi);
    const bool change = plo != 0.0 && phi != 0.0 && (plo > 0.0) != (phi > 0.0);
    for (int it = 0; it < 200 && hi - lo > VP_E_WIDTH * fmax(1.0, fmax(fabs(lo), fabs(hi))); it++) {
      const double mid = 0.5 * (lo + hi);
      if (change) {
        const double pm = vp_horner(S[0], n, mid);
        if (pm == 0.0) { lo = hi = mid; break; }
        if ((pm > 0.0) == (plo > 0.0)) { lo = mid; plo = pm; } else { hi = mid; }
      } else {
        const int vm = vp_sturm_changes(S, deg, ns, mid);
        if (vlo - vm >= 1) hi = mid; else { lo = mid; vlo = vm; }
      }
    }
    double x = 0.5 * (lo + hi);
    for (int it = 0; it < 3; it++) {
      double p = S[0][n], d = 0.0;
      for (int k = n - 1; k >= 0; k--) { d = d * x + p; p = p * x + S[0][k]; }
      if (d == 0.0) break;
      const double y = x - p / d;
      if (!(y >= lo && y <= hi)) break;
      x = y;
    }
    roots[nr++] = x;
  }
  return nr;
}

// The solver's basis of the null space: modified Gram-Schmidt of N0..N3 in order (q0..q3), then the fixed orthogonal
// mix X, Y, Z, W = (q0 - q1 + q2 - q3, q0 + q1 - q2 - q3, q0 - q1 - q2 + q3, q0 + q1 + q2 + q3) / 2, so that no
// chart coordinate is one entry of E (E22, the coordinate of N3, vanishes for small rotations).  false when a vector
// vanishes.
__host__ __device__ inline bool vp_e_basis(double (&N)[4][9])
{
  for (int i = 0; i < 4; i++) {
    for (int j = 0; j < i; j++) {
      double d = 0.0;
      for (int k = 0; k < 9; k++) d += N[i][k] * N[j][k];
      for (int k = 0; k < 9; k++) N[i][k] -= d * N[j][k];
    }
    double n = 0.0;
    for (int k = 0; k < 9; k++) n += N[i][k] * N[i][k];
    if (!(n > 0.0)) return false;
    const double f = 1.0 / sqrt(n);
    for (int k = 0; k < 9; k++) N[i][k] *= f;
  }
  for (int k = 0; k < 9; k++) {
    const double q0 = N[0][k], q1 = N[1][k], q2 = N[2][k], q3 = N[3][k];
    N[0][k] = 0.5 * (q0 - q1 + q2 - q3);
    N[1][k] = 0.5 * (q0 + q1 - q2 - q3);
    N[2][k] = 0.5 * (q0 - q1 - q2 + q3);
    N[3][k] = 0.5 * (q0 + q1 + q2 + q3);
  }
  return true;
}

// Nister's 5-point solver on the basis N (vp_e_basis) of the null space: E = x N0 + y N1 + z N2 + N3.  Row 0 of
// the 10 x 20 system is det E = 0, rows 1 + 3i + j entry (i, j) of 2 E E^T E - tr(E E^T) E = 0.  Gauss-Jordan with
// partial pivoting (the first of equal magnitudes) reduces its first ten columns to the identity; a pivot at or below
// VP_E_PIVOT of the largest |entry| makes the sample degenerate.  Rows 4 - z row 5, 6 - z row 7 and 8 - z row 9 are
// [x y 1] times cubic, cubic, quartic polynomials in z; the determinant of that 3 x 3 polynomial matrix (cofactor
// expansion along its first row) is the degree-10 polynomial, its real roots ascending (vp_real_roots).  For each root,
// (x, y, 1) is the cross product of two rows of the evaluated matrix -- the pair (0,1), (0,2), (1,2) whose third
// component has the largest magnitude, the first of equals -- divided by that component (the root is skipped when it
// is 0).  Returns the number of solutions in E[].
__host__ __device__ inline int vp_five_point(const double (&N)[4][9], double (*E)[9])
{
  double P[9][20];                     // the entries of E, degree-1 polynomials
  for (int k = 0; k < 9; k++) {
    for (int j = 0; j < 20; j++) P[k][j] = 0.0;
    P[k][vp_mono(1, 0, 0)] = N[0][k]; P[k][vp_mono(0, 1, 0)] = N[1][k];
    P[k][vp_mono(0, 0, 1)] = N[2][k]; P[k][vp_mono(0, 0, 0)] = N[3][k];
  }
  double C[10][20];
  for (int r = 0; r < 10; r++)
    for (int j = 0; j < 20; j++) C[r][j] = 0.0;
  {                                    // det E, cofactors along row 0
    double cof[20];
    const int cols[3][2] = {{1, 2}, {0, 2}, {0, 1}};
    const double sg[3] = {1.0, -1.0, 1.0};
    for (int c = 0; c < 3; c++) {
      for (int j = 0; j < 20; j++) cof[j] = 0.0;
      const int a = cols[c][0], b = cols[c][1];
      vp_pmul<1, 1>(P[3 + a], P[6 + b], 1.0, cof);
      vp_pmul<1, 1>(P[3 + b], P[6 + a], -1.0, cof);
      vp_pmul<2, 1>(cof, P[c], sg[c], C[0]);
    }
  }
  {                                    // 2 E E^T E - tr(E E^T) E
    double Q[3][3][20];
    for (int i = 0; i < 3; i++)
      for (int l = i; l < 3; l++) {
        for (int j = 0; j < 20; j++) Q[i][l][j] = 0.0;
        for (int k = 0; k < 3; k++) vp_pmul<1, 1>(P[3 * i + k], P[3 * l + k], 2.0, Q[i][l]);
      }
    double tr[20];
    for (int j = 0; j < 20; j++) tr[j] = 0.5 * (Q[0][0][j] + Q[1][1][j] + Q[2][2][j]);
    for (int i = 0; i < 3; i++) {
      for (int l = 0; l < i; l++)
        for (int j = 0; j < 20; j++) Q[i][l][j] = Q[l][i][j];
      for (int j = 0; j < 20; j++) Q[i][i][j] -= tr[j];
    }
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++)
        for (int l = 0; l < 3; l++) vp_pmul<2, 1>(Q[i][l], P[3 * l + j], 1.0, C[1 + 3 * i + j]);
  }
  double amax = 0.0;
  for (int r = 0; r < 10; r++)
    for (int j = 0; j < 20; j++) amax = fmax(amax, fabs(C[r][j]));
  if (!(amax > 0.0) || !isfinite(amax)) return 0;
#pragma unroll 1
  for (int c = 0; c < 10; c++) {
    int p = c;
    for (int r = c + 1; r < 10; r++)
      if (fabs(C[r][c]) > fabs(C[p][c])) p = r;
    if (!(fabs(C[p][c]) > VP_E_PIVOT * amax)) return 0;
    if (p != c)
      for (int j = c; j < 20; j++) { const double t = C[c][j]; C[c][j] = C[p][j]; C[p][j] = t; }
    const double inv = 1.0 / C[c][c];
    for (int j = c + 1; j < 20; j++) C[c][j] *= inv;
    C[c][c] = 1.0;
    for (int r = 0; r < 10; r++) {
      if (r == c) continue;
      const double f = C[r][c];
      for (int j = c + 1; j < 20; j++) C[r][j] -= f * C[c][j];
      C[r][c] = 0.0;
    }
  }
  // row a - z row b over the last ten columns: x (xz^2 xz x), y (yz^2 yz y) and 1 (z^3 z^2 z 1), ascending in z
  double Bx[3][4], By[3][4], B1[3][5];
  for (int q = 0; q < 3; q++) {
    const double *a = C[4 + 2 * q] + 10, *b = C[5 + 2 * q] + 10;
    Bx[q][0] = a[2]; Bx[q][1] = a[1] - b[2]; Bx[q][2] = a[0] - b[1]; Bx[q][3] = -b[0];
    By[q][0] = a[5]; By[q][1] = a[4] - b[5]; By[q][2] = a[3] - b[4]; By[q][3] = -b[3];
    B1[q][0] = a[9]; B1[q][1] = a[8] - b[9]; B1[q][2] = a[7] - b[8]; B1[q][3] = a[6] - b[7]; B1[q][4] = -b[6];
  }
  double t1[8], t2[8], m1[8], m2[8], m3[7], d[11], e[11];
  vp_upoly_mul(By[1], 3, B1[2], 4, t1);          // ly m1 - l1 my
  vp_upoly_mul(B1[1], 4, By[2], 3, t2);
  for (int k = 0; k < 8; k++) m1[k] = t1[k] - t2[k];
  vp_upoly_mul(Bx[1], 3, B1[2], 4, t1);          // lx m1 - l1 mx
  vp_upoly_mul(B1[1], 4, Bx[2], 3, t2);
  for (int k = 0; k < 8; k++) m2[k] = t1[k] - t2[k];
  vp_upoly_mul(Bx[1], 3, By[2], 3, t1);          // lx my - ly mx
  vp_upoly_mul(By[1], 3, Bx[2], 3, t2);
  for (int k = 0; k < 7; k++) m3[k] = t1[k] - t2[k];
  vp_upoly_mul(Bx[0], 3, m1, 7, d);
  vp_upoly_mul(By[0], 3, m2, 7, e);
  for (int k = 0; k < 11; k++) d[k] -= e[k];
  vp_upoly_mul(B1[0], 4, m3, 6, e);
  for (int k = 0; k < 11; k++) d[k] += e[k];
  double z[10];
  const int nz = vp_real_roots(d, 10, z);
  int ns = 0;
  for (int k = 0; k < nz; k++) {
    double M[3][3];
    for (int q = 0; q < 3; q++) {
      M[q][0] = vp_horner(Bx[q], 3, z[k]); M[q][1] = vp_horner(By[q], 3, z[k]); M[q][2] = vp_horner(B1[q], 4, z[k]);
    }
    const int pr[3][2] = {{0, 1}, {0, 2}, {1, 2}};
    double v[3] = {0.0, 0.0, 0.0};
    for (int q = 0; q < 3; q++) {
      const double *a = M[pr[q][0]], *b = M[pr[q][1]];
      const double w[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
      if (fabs(w[2]) > fabs(v[2])) { v[0] = w[0]; v[1] = w[1]; v[2] = w[2]; }
    }
    if (!(v[2] != 0.0)) continue;
    const double x = v[0] / v[2], y = v[1] / v[2];
    for (int j = 0; j < 9; j++) E[ns][j] = x * N[0][j] + y * N[1][j] + z[k] * N[2][j] + N[3][j];
    ns++;
  }
  return ns;
}

// one thread per sample: 5 draws, calibrated rows, the null space, the 5-point solver; slot sample*10 + r holds the
// r-th solution as Fn = G2^T E G1 (unit norm), NaN when empty
__global__ void __launch_bounds__(VP_HYP_T)
vp_hyp5_kernel(VerifyWave w, int numLoops)
{
  VerifySample h;
  int idx[5];
  if (!vp_hyp_prologue<VP_E_SLOTS>(w, numLoops, h, idx)) return;
  const float4 *__restrict__ xy = h.js.xy;
  const VerifyState *st = h.js.st;
  const VerifyCalib &cal = h.job->cal;
  const double s = st->s;
  double A[5][9], N[4][9];
#pragma unroll
  for (int i = 0; i < 5; i++) {
    const float4 p = xy[idx[i]];
    double x, y, X, Y;
    vp_calibrate(cal.K1, p.x, p.y, x, y);
    vp_calibrate(cal.K2, p.z, p.w, X, Y);
    const double r[9] = {X * x, X * y, X, Y * x, Y * y, Y, x, y, 1};
#pragma unroll
    for (int j = 0; j < 9; j++) A[i][j] = r[j];
  }
  if (!vp_nullspace<5>(A, N) || !vp_e_basis(N)) return;
  double E[VP_E_SLOTS][9];
  const int ne = vp_five_point(N, E);
  double G1[9], G2[9];
  vp_norm_to_calib(cal.K1, st->c1x, st->c1y, s, G1);
  vp_norm_to_calib(cal.K2, st->c2x, st->c2y, s, G2);
  int r = 0;
  for (int k = 0; k < ne; k++) {
    double fn[9];
    vp_sandwich(G2, E[k], G1, fn);
    if (vp_store_unit(h.slot + 9 * r, fn)) r++;
  }
}

// The nearest essential matrix through the eigenvectors of E^T E (Jacobi; descending eigenvalues, the lower index first
// on ties): v1, v2 of the two largest, sigma_i = sqrt(lambda_i), u_i = E v_i / sigma_i, Ep = u1 v1^T + u2 v2^T and
// the right-handed bases u3 = u1 x u2, v3 = v1 x v2 (u[i], v[i] the vectors).  false when sigma2 is not > 0.
__host__ __device__ inline bool vp_essential_project(const double *E, double *Ep, double (&u)[3][3], double (&v)[3][3])
{
  double B[3][3], W[3][3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) B[i][j] = E[i] * E[j] + E[3 + i] * E[3 + j] + E[6 + i] * E[6 + j];
  vp_jacobi<3>(B, W);
  int o[3] = {0, 1, 2};
  for (int i = 1; i < 3; i++)
    for (int j = i; j > 0 && B[o[j]][o[j]] > B[o[j - 1]][o[j - 1]]; j--) { const int t = o[j]; o[j] = o[j - 1]; o[j - 1] = t; }
  for (int a = 0; a < 2; a++) {
    const double sg = sqrt(fmax(B[o[a]][o[a]], 0.0));
    if (!(sg > 0.0) || !isfinite(sg)) return false;
    for (int i = 0; i < 3; i++) v[a][i] = W[i][o[a]];
    for (int i = 0; i < 3; i++) u[a][i] = (E[3 * i] * v[a][0] + E[3 * i + 1] * v[a][1] + E[3 * i + 2] * v[a][2]) / sg;
  }
  u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
  u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
  u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
  v[2][0] = v[0][1] * v[1][2] - v[0][2] * v[1][1];
  v[2][1] = v[0][2] * v[1][0] - v[0][0] * v[1][2];
  v[2][2] = v[0][0] * v[1][1] - v[0][1] * v[1][0];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) Ep[3 * i + j] = u[0][i] * v[0][j] + u[1][i] * v[1][j];
  return true;
}

// (R, t) in front for the calibrated pair (x1, y1) <-> (x2, y2): the least-squares depths of l2 x^2 = l1 R x^1 + t
// are both positive, and the rays are not parallel (sin^2 of their angle above VP_E_PARALLEL)
__host__ __device__ __forceinline__ bool vp_in_front(const double *R, const double *t, double x1, double y1, double x2, double y2)
{
  const double a[3] = {R[0] * x1 + R[1] * y1 + R[2], R[3] * x1 + R[4] * y1 + R[5], R[6] * x1 + R[7] * y1 + R[8]};
  const double b[3] = {x2, y2, 1.0};
  const double aa = a[0] * a[0] + a[1] * a[1] + a[2] * a[2], bb = b[0] * b[0] + b[1] * b[1] + b[2] * b[2];
  const double ab = a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
  const double at = a[0] * t[0] + a[1] * t[1] + a[2] * t[2], bt = b[0] * t[0] + b[1] * t[1] + b[2] * t[2];
  if (!(aa * bb - ab * ab > VP_E_PARALLEL * aa * bb)) return false;
  return ab * bt - at * bb > 0.0 && aa * bt - ab * at > 0.0;      // l1, l2 times the positive determinant
}

// ---- step 7: the refit ---------------------------------------------------------------------------------------------
// rank 2 for F: F (I - v v^T), v the right singular vector of the smallest singular value
__device__ inline void vp_rank2(double (&f)[9])
{
  double B[3][3], W[3][3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) B[i][j] = f[i] * f[j] + f[3 + i] * f[3 + j] + f[6 + i] * f[6 + j];
  vp_jacobi<3>(B, W);
  int l3 = 0;
  for (int i = 1; i < 3; i++) if (B[i][i] < B[l3][l3]) l3 = i;
  const double vv[3] = {W[0][l3], W[1][l3], W[2][l3]};
  for (int r = 0; r < 3; r++) {
    const double fv = f[3 * r] * vv[0] + f[3 * r + 1] * vv[1] + f[3 * r + 2] * vv[2];
    for (int j = 0; j < 3; j++) f[3 * r + j] -= fv * vv[j];
  }
}

// One CTA per job; model is CS_GEOM_HOMOGRAPHY or CS_GEOM_FUNDAMENTAL, or with ESSENTIAL the essential call.  E is an
// instantiation of its own rather than a run-time case, so that F and H keep their register count: at 128 registers
// two CTAs fit an SM and a wave's refits run side by side; E needs more.
//   1. the winning slot's model and its FP32 inliers;
//   2. the normal matrix of their rows (45 upper-triangle entries, fixed-order double reduction): the two DLT rows (H)
//      or the 8-point row (F) on normalised coordinates; for E the 8-point row on calibrated coordinates scaled by
//      lam = s * (K1[0] K1[4] K2[0] K2[4])^(1/4), not centred;
//   3. with at least 4 (H) or 8 (F, E) inliers, its smallest eigenvector f (Jacobi);
//   4. post-processed at unit norm: H as it is; F at rank 2; E = S f S with S = diag(lam, lam, 1), projected to the
//      essential manifold and stored as Fn;
//   5. re-scored, and kept unless it has fewer inliers than the minimal model;
//   6. the final mask (vp_final_mask);
//   7. the output model (pixel coordinates, or E and the pose) and the statistics.
template <bool ESSENTIAL>
__global__ void __launch_bounds__(VP_REFIT_T)
vp_refit_kernel(VerifyWave w, int model)
{
  constexpr bool essential = ESSENTIAL;
  const bool homography = !essential && model == CS_GEOM_HOMOGRAPHY;
  const VerifyJobScratch js = vp_job_scratch(w, blockIdx.x);
  const float4 *__restrict__ xy = js.xy, *__restrict__ un = js.un;
  const double *__restrict__ models = js.models;
  unsigned int *__restrict__ masks = js.masks, *__restrict__ blockCounts = js.counts;
  VerifyState *st = js.st;
  const VerifyCalib &cal = w.jobs[blockIdx.x].cal;
  __shared__ double s_nm[VP_REFIT_T / 32][45];
  __shared__ double s_m[essential ? 3 : 2][9];     // [0] minimal model, [1] refit (E: both as Fn), [2] E: projected E
  __shared__ float s_f[9];
  __shared__ int s_cnt[VP_REFIT_T / 32];
  __shared__ int s_refit;
  const int n = st->numValid;
  const unsigned long long key = st->best;
  const double s = st->s, c1x = st->c1x, c1y = st->c1y, c2x = st->c2x, c2y = st->c2y;
  const float thr2 = st->thr2;
  const int best = key ? (int)~(unsigned int)key : -1;
  int cnt0 = 0, cntR = 0, kept = 0;
  float m[9];
  if (best >= 0) {
    if (threadIdx.x < 9) { s_m[0][threadIdx.x] = models[(size_t)best * 9 + threadIdx.x]; s_f[threadIdx.x] = (float)s_m[0][threadIdx.x]; }
    __syncthreads();
    for (int k = 0; k < 9; k++) m[k] = s_f[k];
    const double lam = essential ? s * sqrt(sqrt(cal.K1[0] * cal.K1[4]) * sqrt(cal.K2[0] * cal.K2[4])) : 0.0;
    double acc[45];
#pragma unroll
    for (int k = 0; k < 45; k++) acc[k] = 0.0;
    int c = 0;
    for (int k = threadIdx.x; k < n; k += VP_REFIT_T) {
      if (!vp_inlier(m, un[k], thr2, homography)) continue;
      c++;
      const float4 p = xy[k];
      double r[2][9];                  // F's zero second row adds exact zeros
      if constexpr (essential) {
        double x, y, X, Y;
        vp_calibrate(cal.K1, p.x, p.y, x, y);
        vp_calibrate(cal.K2, p.z, p.w, X, Y);
        x *= lam; y *= lam; X *= lam; Y *= lam;
        const double r1[9] = {X * x, X * y, X, Y * x, Y * y, Y, x, y, 1};
#pragma unroll
        for (int j = 0; j < 9; j++) r[0][j] = r1[j];
      } else {
        const double x = (p.x - c1x) * s, y = (p.y - c1y) * s, X = (p.z - c2x) * s, Y = (p.w - c2y) * s;
        if (homography) {
          const double r1[9] = {x, y, 1, 0, 0, 0, -X * x, -X * y, -X}, r2[9] = {0, 0, 0, x, y, 1, -Y * x, -Y * y, -Y};
#pragma unroll
          for (int j = 0; j < 9; j++) { r[0][j] = r1[j]; r[1][j] = r2[j]; }
        } else {
          const double r1[9] = {X * x, X * y, X, Y * x, Y * y, Y, x, y, 1};
#pragma unroll
          for (int j = 0; j < 9; j++) { r[0][j] = r1[j]; r[1][j] = 0.0; }
        }
      }
#pragma unroll
      for (int q = 0; q < (essential ? 1 : 2); q++) {
        int e = 0;
#pragma unroll
        for (int i = 0; i < 9; i++)
#pragma unroll
          for (int j = i; j < 9; j++) acc[e++] += r[q][i] * r[q][j];
      }
    }
    vp_warp_normal(acc, s_nm);
    cnt0 = vp_block_count(c, s_cnt);
    if (threadIdx.x == 0) {
      s_refit = 0;
      if (cnt0 >= (homography ? 4 : 8)) {
        double f[9];
        vp_smallest_eigvec(s_nm, f);
        if constexpr (essential) {
          double E[9], u[3][3], v[3][3];
          for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) E[3 * i + j] = f[3 * i + j] * (i < 2 ? lam : 1.0) * (j < 2 ? lam : 1.0);
          if (vp_essential_project(E, s_m[2], u, v)) {
            double G1[9], G2[9], fn[9];
            vp_norm_to_calib(cal.K1, c1x, c1y, s, G1);
            vp_norm_to_calib(cal.K2, c2x, c2y, s, G2);
            vp_sandwich(G2, s_m[2], G1, fn);
            if (vp_store_unit(s_m[1], fn)) s_refit = 1;
          }
        } else {
          if (!homography) vp_rank2(f);
          if (vp_store_unit(s_m[1], f)) s_refit = 1;
        }
      }
    }
    __syncthreads();
    if (s_refit) {
      for (int k = 0; k < 9; k++) m[k] = (float)s_m[1][k];
      int cr = 0;
      for (int k = threadIdx.x; k < n; k += VP_REFIT_T) cr += vp_inlier(m, un[k], thr2, homography);
      cntR = vp_block_count(cr, s_cnt);
      kept = cntR >= cnt0;
    }
    if (!kept)
      for (int k = 0; k < 9; k++) m[k] = s_f[k];
  }
  const int tot = vp_final_mask(best >= 0 ? m : nullptr, un, n, thr2, homography, masks, blockCounts, s_cnt);
  if constexpr (essential) {
    // The final E (the kept refit's projected E, else the one recovered from the winning Fn) projected again with F's
    // output scaling; its four poses R_a = U W V^T, R_b = U W^T V^T and t = +u3, -u3: candidates 0..3 = (R_a, +),
    // (R_a, -), (R_b, +), (R_b, -); the pose with the most final inliers in front (the first of equals).
    __shared__ double s_R[4][9], s_t[4][3];
    __shared__ int s_pose;
    if (threadIdx.x == 0) {
      s_pose = 0;
      double out[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
      if (best >= 0) {
        double E[9], Ep[9], u[3][3], v[3][3];
        if (kept) {
          for (int k = 0; k < 9; k++) E[k] = s_m[2][k];
        } else {
          vp_fn_to_e(cal, *st, s_m[0], E);
        }
        if (vp_essential_project(E, Ep, u, v) && vp_unit_sign(Ep)) {
          for (int k = 0; k < 9; k++) out[k] = Ep[k];
          const double tn = 1.0 / sqrt(u[2][0] * u[2][0] + u[2][1] * u[2][1] + u[2][2] * u[2][2]);
          for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
              const double a = u[1][i] * v[0][j] - u[0][i] * v[1][j], b = u[0][i] * v[1][j] - u[1][i] * v[0][j];
              const double w = u[2][i] * v[2][j];
              s_R[0][3 * i + j] = s_R[1][3 * i + j] = a + w;
              s_R[2][3 * i + j] = s_R[3][3 * i + j] = b + w;
            }
          for (int i = 0; i < 3; i++) {
            s_t[0][i] = s_t[2][i] = u[2][i] * tn;
            s_t[1][i] = s_t[3][i] = -u[2][i] * tn;
          }
          s_pose = 1;
        }
      }
      for (int k = 0; k < 9; k++) st->model[k] = out[k];
    }
    __syncthreads();
    int front[4] = {0, 0, 0, 0};
    if (s_pose) {
      for (int k = threadIdx.x; k < n; k += VP_REFIT_T) {
        if (!((masks[k >> 5] >> (k & 31)) & 1u)) continue;
        const float4 p = xy[k];
        double x, y, X, Y;
        vp_calibrate(cal.K1, p.x, p.y, x, y);
        vp_calibrate(cal.K2, p.z, p.w, X, Y);
        for (int q = 0; q < 4; q++) front[q] += vp_in_front(s_R[q], s_t[q], x, y, X, Y);
      }
      for (int q = 0; q < 4; q++) front[q] = vp_block_count(front[q], s_cnt);
    }
    if (threadIdx.x == 0) {
      int pick = 0, runner = 0;
      for (int q = 1; q < 4; q++) if (front[q] > front[pick]) pick = q;
      for (int q = 0; q < 4; q++) if (q != pick) runner = max(runner, front[q]);
      for (int k = 0; k < 9; k++) st->R[k] = s_pose ? s_R[pick][k] : 0.0;
      for (int k = 0; k < 3; k++) st->t[k] = s_pose ? s_t[pick][k] : 0.0;
      st->pose[0] = front[pick];
      st->pose[1] = runner;
    }
  } else if (threadIdx.x == 0) {
    double out[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (best >= 0) vp_denormalise(kept ? s_m[1] : s_m[0], model, c1x, c1y, c2x, c2y, s, out);
    for (int k = 0; k < 9; k++) st->model[k] = out[k];
  }
  if (threadIdx.x == 0) {
    st->total = tot;
    st->stats[0] = n;
    st->stats[2] = (long long)st->samples;
    st->stats[3] = (long long)st->models;
    st->stats[4] = best;
    st->stats[5] = cnt0;
    st->stats[6] = kept;
    st->stats[7] = tot;
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------
// model slots per sample: up to 3 roots of the 7-point cubic (F; H uses the first), up to 10 of the 5-point solver (E)
static int vp_slots_per_sample(int model) { return model == VERIFY_ESSENTIAL ? VP_E_SLOTS : 3; }

// The waves of a batch, a job's extent being its row CTAs; a slot is 9 doubles and a count.
static WavePlan verify_plan(const cs_verify_job *jobs, int numJobs, int numLoops, int model)
{
  const size_t slotBytes = (size_t)vp_slots_per_sample(model) * numLoops * (9 * sizeof(double) + sizeof(unsigned int));
  return wave_plan(jobs, numJobs, slotBytes, [](const cs_verify_job &a) { return (size_t)list_ctas(a.numPairs); });
}

struct VerifyLayout {
  size_t jobs, masks, counts, xy, un, orig, models, slotCounts, state, bytes;
};

// The device table of the batch's non-empty jobs, then the scratch of one wave (reused by the next).
static VerifyLayout verify_layout(const WavePlan &p, int numLoops, int model)
{
  VerifyLayout L;
  Layout o(256);
  const size_t live = std::max(p.live.size(), (size_t)1), J = std::min(live, (size_t)p.perWave);
  const size_t P = std::max(p.extent, (size_t)1) * LIST_ROWS, S = vp_slots_per_sample(model) * (size_t)numLoops * J;
  L.jobs = o.take(live * sizeof(VerifyJob));
  L.masks = o.take(P / 32 * sizeof(unsigned int));
  L.counts = o.take(P / LIST_ROWS * sizeof(unsigned int));
  L.xy = o.take(P * sizeof(float4));
  L.un = o.take(P * sizeof(float4));
  L.orig = o.take(P * sizeof(int));
  L.models = o.take(S * 9 * sizeof(double));
  L.slotCounts = o.take(S * sizeof(unsigned int));
  L.state = o.take(J * sizeof(VerifyState));
  L.bytes = o.bytes;
  return L;
}

// Per wave: steps 1-4 (and, with full, 5-8) on the stream, then the wave's states copied to the pinned area.
// full == false stops after scoring (the models and counts of the last wave stay in scratch).
int verify_enqueue(DeviceCtx &c, const cs_verify_job *jobs, int numJobs, const VerifyCalib *cal, int model, int numLoops,
                   float thresh, bool full)
{
  const WavePlan plan = verify_plan(jobs, numJobs, numLoops, model);
  const int live = (int)plan.live.size();
  if (live == 0) return 0;
  const VerifyLayout L = verify_layout(plan, numLoops, model);
  int r;
  if ((r = c.verify.grow(L.bytes)) < 0) return r;
  VerifyState *h_states;
  VerifyJob *h_jobs;
  if ((r = pinned_states_and_jobs(c.h_verify, live, h_states, h_jobs)) < 0) return r;
  char *b = c.verify.as<char>();
  const cudaStream_t st = c.stream;
  const bool essential = model == VERIFY_ESSENTIAL;
  const int perSample = vp_slots_per_sample(model), slots = perSample * numLoops;
  // the table; the row and score bases count from the first job of each wave
  int rowBase = 0, scoreBase = 0;
  for (int q = 0; q < live; q++) {
    if (q % plan.perWave == 0) rowBase = scoreBase = 0;
    const cs_verify_job &a = jobs[plan.live[q]];
    VerifyJob &t = h_jobs[q];
    t.s1 = static_cast<const SiftPoint *>(a.s1);
    t.s2 = static_cast<const SiftPoint *>(a.s2);
    t.pairs = reinterpret_cast<const int2 *>(a.pairs);
    t.inliers = reinterpret_cast<int2 *>(a.inliers);
    t.seed = a.seed;
    t.n1 = a.n1; t.n2 = a.n2; t.numPairs = a.numPairs; t.maxInliers = a.maxInliers;
    t.rowBase = rowBase;
    t.scoreBase = scoreBase;
    t.cal = cal ? cal[plan.live[q]] : VerifyCalib{};
    rowBase += list_ctas(a.numPairs);
    scoreBase += idivup(a.numPairs, VP_CHUNK);
  }
  VerifyJob *d_jobs = reinterpret_cast<VerifyJob *>(b + L.jobs);
  CS_CUDA(cudaMemcpyAsync(d_jobs, h_jobs, (size_t)live * sizeof(VerifyJob), cudaMemcpyHostToDevice, st));
  VerifyWave w;
  w.slots = slots;
  w.masks = reinterpret_cast<unsigned int *>(b + L.masks);
  w.counts = reinterpret_cast<unsigned int *>(b + L.counts);
  w.xy = reinterpret_cast<float4 *>(b + L.xy);
  w.un = reinterpret_cast<float4 *>(b + L.un);
  w.orig = reinterpret_cast<int *>(b + L.orig);
  w.models = reinterpret_cast<double *>(b + L.models);
  w.slotCounts = reinterpret_cast<unsigned int *>(b + L.slotCounts);
  w.st = reinterpret_cast<VerifyState *>(b + L.state);
  const int hypPerJob = idivup(numLoops, VP_HYP_T), argPerJob = idivup(slots, 256);
  const int scoreModel = essential ? CS_GEOM_FUNDAMENTAL : model;      // E is scored as its Fn
  const int modelBlocks = idivup(model == CS_GEOM_HOMOGRAPHY ? numLoops : slots, VP_SC_T);
  cudaEvent_t *tev = full ? match_timing_events() : nullptr;
  for (int q0 = 0; q0 < live; q0 += plan.perWave) {
    const int nj = std::min(plan.perWave, live - q0);
    const VerifyJob &last = h_jobs[q0 + nj - 1];
    const int rows = last.rowBase + list_ctas(last.numPairs);
    const int chunks = last.scoreBase + idivup(last.numPairs, VP_CHUNK);
    w.jobs = d_jobs + q0;
    w.numJobs = nj;
    if (tev) cudaEventRecord(tev[0], st);
    vp_flags_kernel<<<rows, LIST_ROWS, 0, st>>>(w);
    if (tev) cudaEventRecord(tev[1], st);
    vp_compact_kernel<<<rows, LIST_ROWS, 0, st>>>(w);
    if (tev) cudaEventRecord(tev[2], st);
    vp_norm_kernel<<<nj, 1024, 0, st>>>(w, thresh);
    if (tev) cudaEventRecord(tev[3], st);
    if (essential)
      vp_hyp5_kernel<<<nj * hypPerJob, VP_HYP_T, 0, st>>>(w, numLoops);
    else
      vp_hyp_kernel<<<nj * hypPerJob, VP_HYP_T, 0, st>>>(w, numLoops, model);
    if (tev) cudaEventRecord(tev[4], st);
    vp_score_kernel<<<dim3(chunks, modelBlocks), VP_SC_T, 0, st>>>(w, scoreModel);
    count_launch(5);
    if (full) {
      if (tev) cudaEventRecord(tev[5], st);
      vp_argmax_kernel<<<nj * argPerJob, 256, 0, st>>>(w, perSample);
      if (tev) cudaEventRecord(tev[6], st);
      if (essential)
        vp_refit_kernel<true><<<nj, VP_REFIT_T, 0, st>>>(w, model);
      else
        vp_refit_kernel<false><<<nj, VP_REFIT_T, 0, st>>>(w, model);
      if (tev) cudaEventRecord(tev[7], st);
      vp_write_kernel<<<rows, LIST_ROWS, 0, st>>>(w);
      if (tev) cudaEventRecord(tev[8], st);
      count_launch(3);
    }
    CS_CUDA(cudaGetLastError());
    CS_CUDA(cudaMemcpyAsync(h_states + q0, w.st, (size_t)nj * sizeof(VerifyState), cudaMemcpyDeviceToHost, st));
    if (tev) {
      static const char *const stages[] = {"flags", "compact", "norm", "hyp", "score", "argmax", "refit", "write"};
      int pairs = 0;
      for (int q = q0; q < q0 + nj; q++) pairs += h_jobs[q].numPairs;
      report_stage_times(tev, stages, 8, "verify timing model=%d pairs=%d loops=%d", model, pairs, numLoops);
    }
  }
  return 0;
}

// After verify_enqueue and a synchronize: the q-th non-empty job's count, model and statistics from its copied state.
int verify_result(const DeviceCtx &c, int q, int numPairs, double model_out[9], long long stats[8])
{
  const VerifyState *v = c.h_verify.as<const VerifyState>() + q;
  for (int k = 0; k < 9; k++) model_out[k] = v->model[k];
  for (int k = 0; k < 8; k++) stats[k] = v->stats[k];
  stats[1] = (long long)numPairs - v->numValid;
  return v->total;
}

// The same after an essential launch: E (in model), the pose and the ten statistics.
int verify_essential_result(const DeviceCtx &c, int q, int numPairs, double E[9], double R[9], double t[3],
                            long long stats[10])
{
  const VerifyState *v = c.h_verify.as<const VerifyState>() + q;
  for (int k = 0; k < 9; k++) R[k] = v->R[k];
  for (int k = 0; k < 3; k++) t[k] = v->t[k];
  stats[8] = v->pose[0];
  stats[9] = v->pose[1];
  return verify_result(c, q, numPairs, E, stats);
}

// After verify_enqueue(full = false) of one job: every slot's model in pixel coordinates (NaN-filled when empty), every
// slot's inlier count and the normalisation {c1x, c1y, c2x, c2y, s} (synchronizes).  Returns the number of valid pairs.
// An essential slot's Fn becomes E = (T2 K2)^T Fn (T1 K1) with F's output scaling.
int verify_models_to_host(DeviceCtx &c, const cs_verify_job &job, int numLoops, int model, const VerifyCalib *cal,
                          double *h_models, int *h_counts, double h_norm[5])
{
  const VerifyLayout L = verify_layout(verify_plan(&job, 1, numLoops, model), numLoops, model);
  const char *b = c.verify.as<const char>();
  const size_t S = vp_slots_per_sample(model) * (size_t)numLoops;
  CS_CUDA(cudaMemcpyAsync(h_models, b + L.models, S * 9 * sizeof(double), cudaMemcpyDeviceToHost, c.stream));
  CS_CUDA(cudaMemcpyAsync(h_counts, b + L.slotCounts, S * sizeof(int), cudaMemcpyDeviceToHost, c.stream));
  CS_CUDA(cudaStreamSynchronize(c.stream));
  const VerifyState *v = c.h_verify.as<const VerifyState>();
  h_norm[0] = v->c1x; h_norm[1] = v->c1y; h_norm[2] = v->c2x; h_norm[3] = v->c2y; h_norm[4] = v->s;
  for (size_t k = 0; k < S; k++) {
    double *m = h_models + 9 * k;
    if (std::isnan(m[0])) { for (int j = 0; j < 9; j++) m[j] = NAN; continue; }
    double out[9];
    if (model == VERIFY_ESSENTIAL) {
      vp_fn_to_e(*cal, *v, m, out);
      vp_unit_sign(out);
    } else {
      vp_denormalise(m, model, v->c1x, v->c1y, v->c2x, v->c2y, v->s, out);
    }
    for (int j = 0; j < 9; j++) m[j] = out[j];
  }
  return v->numValid;
}

}  // namespace cs
