// triangulate.cu -- triangulation of feature tracks with known cameras (cs_triangulate_tracks).  The rules (validity,
// hypotheses, admissibility, inliers, winner, refit, outputs) are stated in cudasift_b200.h at cs_triangulate_tracks;
// tests/triangulate_oracle.py restates them in float64.
//
// One launch.  A warp owns a track at a time; the warps of a grid of one resident wave claim tracks from one queue
// (the first track of a warp is its global warp index, the next ones come from a counter zeroed before the launch), so
// a long track occupies one warp while the others go on.  Per track:
//   1. the valid members, compacted in member order by ballots: rank r < TR_CAP in the warp's shared memory, the rest
//      in global scratch at offsets[k] + r; the member outputs of invalid members are written here
//   2. lane l evaluates hypotheses l, l + 32, ...: the two-view DLT through the 4x4 normal matrix and vp_jacobi<4> in
//      FP64 registers, the admissibility tests, then the inlier count over every valid member (the member reads are the
//      same address in every lane of the loop: broadcasts)
//   3. the winner: a butterfly max over the packed key (count + 1) << 32 | ~h, so the most inliers, then the lowest h;
//      its point comes from lane h & 31
//   4. the refit: each lane sums the DLT rows of the winner's inliers among ranks lane, lane + 32, ... in rank order, a
//      fixed xor butterfly adds the ten sums (a + b and b + a round alike, so every lane holds the same bits), and every
//      lane runs the same Jacobi; its inliers are counted with the same test
//   5. the point, the count and, per valid member, the error and the inlier byte
// Nothing depends on scheduling: a track's arithmetic is a fixed sequence whichever warp runs it, and the statistics are
// integer sums (warp butterflies, then one atomicAdd per warp and field).
#include <algorithm>
#include <cmath>
#include <math_constants.h>

#include "common.cuh"
#include "vp_math.cuh"

namespace cs {

namespace {

constexpr int TR_THREADS = 128;
constexpr int TR_WARPS = TR_THREADS / 32;
constexpr int TR_CAP = 128;          // valid members per warp staged in shared memory (16 bytes each)
constexpr int TR_DRAWS = 16;         // draws per sample before it is degenerate

// One image as the kernel reads it (built on the host in double from K, R and t).
struct TrCam {
  double P[12];                      // K [R | t], row-major 3 x 4: world point -> homogeneous pixel
  double Rt[12];                     // [R | t]: world point -> camera; the DLT rows and the depth use it
  double K[6];                       // K[0..5] (vp_calibrate reads 0, 1, 2, 4 and 5)
  double C[3];                       // the centre -R^T t
  const SiftPoint *pts;
  int n, pad;
};

// A valid member: its pixel coordinates, image and position in d_members.
struct TrEntry {
  float x, y;
  int a, pos;
};

struct TrParams {
  const TrCam *cams;
  const int *offsets;
  const int2 *members;
  TrEntry *spill;                    // [numMembers]: valid members of rank >= TR_CAP, at offsets[k] + rank
  double *points;
  int *counts;
  float *errors;
  unsigned char *inlier;
  unsigned long long *stats;         // the eight statistics of cs_triangulate_tracks
  unsigned int *queue;               // tracks claimed past the first wave
  unsigned long long seed;
  double thr2, cosMin;               // maxError^2, cos(minTriAngle)
  int numImages, numTracks, numMembers, numTrials;
};

__device__ __forceinline__ TrEntry tr_entry(const TrEntry *s_e, const TrEntry *spill, int lo, int r)
{
  return r < TR_CAP ? s_e[r] : spill[lo + r];
}

// The ranks (p, q), p < q, of exhaustive hypothesis h: the pairs in lexicographic order.
__device__ __forceinline__ void tr_pair(int h, int V, int &p, int &q)
{
  p = 0;
  while (h >= V - 1 - p) {
    h -= V - 1 - p;
    p++;
  }
  q = p + 1 + h;
}

// The two ranks of sample s of track k (the header's sampler); false when 16 draws give fewer than two distinct ranks.
__device__ __forceinline__ bool tr_draw(unsigned long long seed, int k, int s, int V, int &p, int &q)
{
  int got = 0;
  for (int d = 0; d < TR_DRAWS && got < 2; d++) {
    const unsigned long long x = vp_splitmix64(
        seed + 0x9E3779B97F4A7C15ull * (((unsigned long long)k << 24) | ((unsigned long long)s << 4) | (unsigned)d));
    const int i = (int)(((x >> 32) * (unsigned long long)V) >> 32);
    if (got == 0) { p = i; got = 1; }
    else if (i != p) { q = i; got = 2; }
  }
  return got == 2;
}

// The member's two DLT rows x^ P[2] - P[0] and y^ P[2] - P[1] (P = [R | t], calibrated coordinates) added to the
// normal matrix's ten sums (00 01 02 03 11 12 13 22 23 33), first row first.
__device__ __forceinline__ void tr_add_rows(const TrCam &c, float x, float y, double (&s)[10])
{
  double cx, cy;
  vp_calibrate(c.K, (double)x, (double)y, cx, cy);
  const double w[2] = {cx, cy};
#pragma unroll
  for (int r = 0; r < 2; r++) {
    double row[4];
#pragma unroll
    for (int j = 0; j < 4; j++) row[j] = w[r] * c.Rt[8 + j] - c.Rt[4 * r + j];
    int k = 0;
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int j = i; j < 4; j++) s[k++] += row[i] * row[j];
  }
}

// The eigenvector of the smallest eigenvalue of the normal matrix (the lowest index on ties), dehomogenised; false when
// its w is 0 or the point is not finite.
__device__ __forceinline__ bool tr_solve(const double (&s)[10], double (&X)[3])
{
  double A[4][4] = {{s[0], s[1], s[2], s[3]}, {s[1], s[4], s[5], s[6]}, {s[2], s[5], s[7], s[8]},
                    {s[3], s[6], s[8], s[9]}};
  double V[4][4];
  vp_jacobi<4>(A, V);
  double best = A[0][0], h[4] = {V[0][0], V[1][0], V[2][0], V[3][0]};
#pragma unroll
  for (int j = 1; j < 4; j++)
    if (A[j][j] < best) {
      best = A[j][j];
#pragma unroll
      for (int i = 0; i < 4; i++) h[i] = V[i][j];
    }
  if (h[3] == 0.0) return false;
#pragma unroll
  for (int i = 0; i < 3; i++) X[i] = h[i] / h[3];
  return isfinite(X[0]) && isfinite(X[1]) && isfinite(X[2]);
}

// tr_member (the member rule), tr_inlier (the reprojection inlier rule) and tr_reproject (the member outputs) are in
// vp_math.cuh.
__device__ __forceinline__ double tr_depth(const TrCam &c, const double (&X)[3])
{
  return c.Rt[8] * X[0] + c.Rt[9] * X[1] + c.Rt[10] * X[2] + c.Rt[11];
}

__global__ void __launch_bounds__(TR_THREADS) triangulate_kernel(TrParams p)
{
  __shared__ TrEntry s_all[TR_WARPS][TR_CAP];
  const unsigned full = 0xffffffffu;
  const int lane = (int)threadIdx.x & 31, warp = (int)threadIdx.x >> 5;
  const int totalWarps = (int)gridDim.x * TR_WARPS;
  __shared__ unsigned long long s_st[8];                   // the CTA's statistics
  TrEntry *s_e = s_all[warp];
  if (threadIdx.x < 8) s_st[threadIdx.x] = 0;
  __syncthreads();

  for (int k = (int)blockIdx.x * TR_WARPS + warp;;) {
    if (k >= p.numTracks) break;
    const int lo = p.offsets[k], hi = p.offsets[k + 1];
    if (lo < 0 || hi < lo || hi > p.numMembers) {             // malformed: no point, no member output
      if (lane == 0) {
        atomicAdd(&s_st[1], 1ull);
#pragma unroll
        for (int i = 0; i < 3; i++) p.points[3 * (size_t)k + i] = CUDART_NAN;
        p.counts[k] = 0;
      }
    } else {
      // 1. the valid members in member order
      int V = 0, invalid = 0, evaluated = 0, admissible = 0;   // the last three: this lane's share
      for (int b = lo; b < hi; b += 32) {
        const int m = b + lane;
        bool ok = false;
        TrEntry e{0.0f, 0.0f, 0, m};
        if (m < hi) {
          const int2 af = p.members[m];
          ok = tr_member(p.cams, p.numImages, af, e.x, e.y);
          if (ok) e.a = af.x;
          if (!ok) {
            invalid++;
            if (p.errors) p.errors[m] = CUDART_NAN_F;
            if (p.inlier) p.inlier[m] = 0;
          }
        }
        const unsigned bal = __ballot_sync(full, ok);
        if (ok) {
          const int r = V + __popc(bal & ((1u << lane) - 1u));
          if (r < TR_CAP) s_e[r] = e; else p.spill[lo + r] = e;
        }
        V += __popc(bal);
      }
      __syncwarp();

      // 2. the hypotheses, lane-strided
      const long long numPairs = (long long)V * (V - 1) / 2;
      const bool exhaustive = numPairs <= p.numTrials;
      const int H = V < 2 ? 0 : exhaustive ? (int)numPairs : p.numTrials;
      unsigned long long key = 0;                             // this lane's best: (count + 1) << 32 | ~h, 0 = none
      double X[3] = {0.0, 0.0, 0.0};
      for (int h = lane; h < H; h += 32) {
        int r0 = 0, r1 = 0;
        if (exhaustive) tr_pair(h, V, r0, r1);
        else if (!tr_draw(p.seed, k, h, V, r0, r1)) continue;
        evaluated++;
        const TrEntry e0 = tr_entry(s_e, p.spill, lo, r0), e1 = tr_entry(s_e, p.spill, lo, r1);
        if (e0.a == e1.a) continue;
        const TrCam &c0 = p.cams[e0.a], &c1 = p.cams[e1.a];
        double s[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0}, Y[3];
        tr_add_rows(c0, e0.x, e0.y, s);
        tr_add_rows(c1, e1.x, e1.y, s);
        if (!tr_solve(s, Y)) continue;
        if (!(tr_depth(c0, Y) > 0.0) || !(tr_depth(c1, Y) > 0.0)) continue;
        double ab = 0.0, aa = 0.0, bb = 0.0;
#pragma unroll
        for (int i = 0; i < 3; i++) {
          const double a = Y[i] - c0.C[i], b = Y[i] - c1.C[i];
          ab += a * b; aa += a * a; bb += b * b;
        }
        if (!(ab <= p.cosMin * sqrt(aa * bb))) continue;
        admissible++;
        int cnt = 0;
        for (int r = 0; r < V; r++) {
          const TrEntry e = tr_entry(s_e, p.spill, lo, r);
          cnt += tr_inlier(p.cams[e.a].P, Y, e.x, e.y, p.thr2);
        }
        const unsigned long long kk = ((unsigned long long)(cnt + 1) << 32) | (0xffffffffu - (unsigned)h);
        if (kk > key) {
          key = kk;
#pragma unroll
          for (int i = 0; i < 3; i++) X[i] = Y[i];
        }
      }

      // 3. the winner
      const unsigned long long best = vp_warp_max(key);
      const int src = (int)((0xffffffffu - (unsigned)best) & 31u);
#pragma unroll
      for (int i = 0; i < 3; i++) X[i] = __shfl_sync(full, X[i], src);
      int count = best ? (int)(best >> 32) - 1 : 0;

      // 4. the refit over the winner's inliers
      bool kept = false;
      if (best && count >= 2) {
        double s[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0}, Y[3];
        for (int r = lane; r < V; r += 32) {
          const TrEntry e = tr_entry(s_e, p.spill, lo, r);
          const TrCam &c = p.cams[e.a];
          if (tr_inlier(c.P, X, e.x, e.y, p.thr2)) tr_add_rows(c, e.x, e.y, s);
        }
        vp_warp_sum(s);
        const bool finite = tr_solve(s, Y);
        int cnt = 0;
        if (finite)
          for (int r = lane; r < V; r += 32) {
            const TrEntry e = tr_entry(s_e, p.spill, lo, r);
            cnt += tr_inlier(p.cams[e.a].P, Y, e.x, e.y, p.thr2);
          }
        cnt = __reduce_add_sync(full, cnt);
        if (finite && cnt >= count) {
          kept = true;
          count = cnt;
#pragma unroll
          for (int i = 0; i < 3; i++) X[i] = Y[i];
        }
      }

      // 5. the outputs
      const bool has = best && count >= 2;
      invalid = __reduce_add_sync(full, invalid);
      evaluated = __reduce_add_sync(full, evaluated);
      admissible = __reduce_add_sync(full, admissible);
      if (lane == 0) {
        atomicAdd(&s_st[0], 1ull);
        if (invalid) atomicAdd(&s_st[2], (unsigned long long)invalid);
        if (evaluated) atomicAdd(&s_st[3], (unsigned long long)evaluated);
        if (admissible) atomicAdd(&s_st[4], (unsigned long long)admissible);
        if (has) {
          atomicAdd(&s_st[5], 1ull);
          if (kept) atomicAdd(&s_st[6], 1ull);
          atomicAdd(&s_st[7], (unsigned long long)count);
        }
#pragma unroll
        for (int i = 0; i < 3; i++) p.points[3 * (size_t)k + i] = has ? X[i] : CUDART_NAN;
        p.counts[k] = has ? count : 0;
      }
      if (p.errors || p.inlier)
        for (int r = lane; r < V; r += 32) {
          const TrEntry e = tr_entry(s_e, p.spill, lo, r);
          float err = CUDART_NAN_F;
          unsigned char in = 0;
          if (has) tr_reproject(p.cams[e.a].P, X, e.x, e.y, p.thr2, err, in);
          if (p.errors) p.errors[e.pos] = err;
          if (p.inlier) p.inlier[e.pos] = in;
        }
      __syncwarp();                                           // the staged members are read before the next track
    }
    int next = 0;
    if (lane == 0) next = totalWarps + (int)atomicAdd(p.queue, 1u);
    k = __shfl_sync(full, next, 0);
  }

  __syncthreads();
  if (threadIdx.x < 8 && s_st[threadIdx.x]) atomicAdd(&p.stats[threadIdx.x], s_st[threadIdx.x]);
}

}  // namespace

int triangulate_enqueue(DeviceCtx &c, const cs_match_set *sets, int numImages, const double *Ks, const double *Rs,
                        const double *ts, const int *offsets, int numTracks, const int *members, int numMembers,
                        int numTrials, double maxError, double minTriAngle, unsigned long long seed, double *points,
                        int *counts, float *errors, unsigned char *inlier)
{
  // scratch: the statistics and the queue word, the camera table, the spilled members
  Layout L(256);
  const size_t statsAt = L.take(8 * sizeof(unsigned long long) + sizeof(unsigned int));
  const size_t camAt = L.take((size_t)numImages * sizeof(TrCam)), spillAt = L.bytes;
  int r = c.tri.grow(spillAt + (size_t)numMembers * sizeof(TrEntry));
  if (r < 0) return r;
  char *base = c.tri.as<char>();

  // the camera table is built in pinned memory after the statistics' landing area (the previous call ended in a
  // synchronize) and goes up in one copy
  if ((r = c.h_tri.grow(spillAt)) < 0) return r;
  TrCam *cams = reinterpret_cast<TrCam *>(c.h_tri.as<char>() + camAt);
  for (int a = 0; a < numImages; a++) {
    TrCam &m = cams[a];
    const double *K = Ks + 9 * (size_t)a, *R = Rs + 9 * (size_t)a, *t = ts + 3 * (size_t)a;
    for (int i = 0; i < 3; i++) {
      for (int j = 0; j < 3; j++) m.Rt[4 * i + j] = R[3 * i + j];
      m.Rt[4 * i + 3] = t[i];
    }
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 4; j++)
        m.P[4 * i + j] = K[3 * i] * m.Rt[j] + K[3 * i + 1] * m.Rt[4 + j] + K[3 * i + 2] * m.Rt[8 + j];
    for (int i = 0; i < 6; i++) m.K[i] = K[i];
    for (int i = 0; i < 3; i++) m.C[i] = -(R[i] * t[0] + R[3 + i] * t[1] + R[6 + i] * t[2]);
    m.pts = static_cast<const SiftPoint *>(sets[a].pts);
    m.n = sets[a].n;
    m.pad = 0;
  }

  TrParams prm;
  prm.stats = reinterpret_cast<unsigned long long *>(base + statsAt);
  prm.queue = reinterpret_cast<unsigned int *>(prm.stats + 8);
  prm.cams = reinterpret_cast<const TrCam *>(base + camAt);
  prm.spill = reinterpret_cast<TrEntry *>(base + spillAt);
  prm.offsets = offsets;
  prm.members = reinterpret_cast<const int2 *>(members);
  prm.points = points;
  prm.counts = counts;
  prm.errors = errors;
  prm.inlier = inlier;
  prm.seed = seed;
  prm.thr2 = maxError * maxError;
  prm.cosMin = cos(minTriAngle * (M_PI / 180.0));
  prm.numImages = numImages;
  prm.numTracks = numTracks;
  prm.numMembers = numMembers;
  prm.numTrials = numTrials;

  const int wave = resident_grid<triangulate_kernel, TR_THREADS>();
  if (wave < 0) return wave;
  const int grid = std::min(wave, idivup(numTracks, TR_WARPS));
  const cudaStream_t st = c.stream;
  CS_CUDA(cudaMemsetAsync(base + statsAt, 0, camAt - statsAt, st));
  if (numImages) CS_CUDA(cudaMemcpyAsync(base + camAt, cams, (size_t)numImages * sizeof(TrCam), cudaMemcpyHostToDevice, st));
  triangulate_kernel<<<grid, TR_THREADS, 0, st>>>(prm);
  count_launch();
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaMemcpyAsync(c.h_tri.p, prm.stats, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  return 0;
}

}  // namespace cs
