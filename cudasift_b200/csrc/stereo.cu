// stereo.cu -- dense reconstruction: undistorted images (cs_undistort_images), PatchMatch stereo with red-black
// propagation (cs_patch_match_stereo), its geometric-consistency pass (cs_patch_match_stereo_geometric) and the fusion
// of depth maps (cs_fuse_depth_maps).  The header states every rule; tests/stereo_oracle.py and
// tests/stereo_geom_oracle.py restate them in float64.
//
// A half-step reads the other colour and the pixel's own state only, and writes the pixel's own state, so the maps are
// the state and no pixel's result depends on the order in which threads run.  The geometric pass also reads the
// sources' prior maps, which are inputs of the call and never written.  The only atomics are integer counts.
#include "common.cuh"
#include "ordered_list.cuh"
#include "vp_math.cuh"

namespace cs {

namespace {

constexpr int ST_THREADS = 128;
constexpr int ST_MAX_SOURCES = 32;
constexpr float ST_VAR_FLOOR = 1.0f;

struct StImage {
  const float *img;
  int w, h, pitch;
  int job;                // the job whose ref this image is, or -1
  double K[9], Kinv[9], R[9], t[3];
};

struct StSrc {
  int image;
  float A[9], b[3];
};

struct StJob {
  int ref, w, h;
  int src0, numSources;
  float dmin, dmax;
  double Kinv[9];
  float *depth, *normal, *cost;
  long long all0, half0;  // first thread of the job in the full-image and half-step grids
};

// The per-job counters of a call: pixels (host), invalid view evaluations, pixels whose final cost is 2.
struct StCounts {
  unsigned long long v[3];
};
// The geometric pass's table per source (parallel to the StSrc table): R_sr, t_sr in float64 and the source's prior
// depth map (NULL: no prior) with its size.
struct StGeo {
  double R[9], t[3];
  const float *depth;
  int w, h;
};

// The geometric pass's prior of a job's ref.
struct StPrior {
  const float *depth, *normal;
};

// the scratch the header states
static_assert(sizeof(StImage) == 264 && sizeof(StJob) == 144 && sizeof(StSrc) == 52 && sizeof(StCounts) == 24,
              "stereo table sizes");
static_assert(sizeof(StGeo) == 112 && sizeof(StPrior) == 16, "geometric table sizes");

// The draws of the geometric pass use counter iterations 32 (start) and 32 + k (iteration k <= 31), apart from the
// photometric pass's 0 .. 32 under the same seed.
constexpr int ST_GEOM_IT0 = 32;

__device__ __forceinline__ float st_bilinear(const float *__restrict__ img, int w, int h, int pitch, float u, float v)
{
  u = fminf(fmaxf(u, 0.0f), (float)(w - 1));
  v = fminf(fmaxf(v, 0.0f), (float)(h - 1));
  const int x0 = min((int)u, w - 2), y0 = min((int)v, h - 2);
  const float fx = u - (float)x0, fy = v - (float)y0;
  const float *r0 = img + (size_t)y0 * pitch + x0, *r1 = r0 + pitch;
  const float i00 = __ldg(r0), i10 = __ldg(r0 + 1), i01 = __ldg(r1), i11 = __ldg(r1 + 1);
  const float a = fmaf(fx, i10 - i00, i00), b = fmaf(fx, i11 - i01, i01);
  return fmaf(fy, b - a, a);
}

// ---- undistortion ---------------------------------------------------------------------------------------------------

struct UdImage {
  const float *img;
  float *out;
  int w, h, pitch;
  double K[9], k1, k2;
};

// A 32 x 8 tile of image z for z = blockIdx.z, blockIdx.z + gridDim.z, ... (gridDim.z is at most 65535).
__global__ void __launch_bounds__(256) undistort_images_kernel(const UdImage *__restrict__ ims, int numImages,
                                                               unsigned long long *__restrict__ outside)
{
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  for (int z = blockIdx.z; z < numImages; z += gridDim.z) {
    const UdImage &m = ims[z];
    bool out = false;
    if (x < m.w && y < m.h) {
      const double *K = m.K;
      const double b = (y - K[5]) / K[4], a = (x - K[2] - K[1] * b) / K[0];
      const double r2 = a * a + b * b, s = 1.0 + m.k1 * r2 + m.k2 * r2 * r2;
      const float u = (float)(K[0] * a * s + K[1] * b * s + K[2]), v = (float)(K[4] * b * s + K[5]);
      out = !(u >= 0.0f && u <= (float)(m.w - 1) && v >= 0.0f && v <= (float)(m.h - 1));
      m.out[(size_t)y * m.w + x] = out ? 0.0f : st_bilinear(m.img, m.w, m.h, m.pitch, u, v);
    }
    const unsigned int n = __popc(__ballot_sync(0xffffffffu, out));
    if ((threadIdx.x & 31) == 0 && n) atomicAdd(outside + z, (unsigned long long)n);
  }
}

// ---- PatchMatch -----------------------------------------------------------------------------------------------------

struct PmParams {
  const StImage *images;
  const StJob *jobs;
  const StSrc *srcs;
  StCounts *counts;
  int numJobs;
  int radius, step, topK;
  unsigned long long seed;
  int iteration, colour;   // the half-step's iteration (1..) and colour (0 even, 1 odd)
};

// The geometric pass's own parameters: a kernel argument after PmParams and the total, so the photometric kernels'
// arguments keep their offsets.
struct PmGeom {
  const StGeo *geo;        // per source, parallel to srcs
  const StPrior *priors;   // per job
  StCounts *counts;        // per job: {valid view evaluations capped at gmax, pixels started from a draw, 0}
  float lambda;
  double gmax;
};

struct Hyp {
  float z, n[3];
};

__device__ __forceinline__ double st_draw(unsigned long long seed, const StJob &J, int x, int y, int iteration, int slot)
{
  const unsigned long long c =
      ((((unsigned long long)J.ref << 24) + (unsigned long long)(y * J.w + x)) * 64 + iteration) * 16 + slot;
  return (double)(vp_splitmix64(seed + 0x9E3779B97F4A7C15ull * c) >> 11) * 0x1.0p-53;
}

__device__ __forceinline__ void st_ray(const double *Ki, int x, int y, double (&r)[3])
{
  for (int k = 0; k < 3; k++) r[k] = Ki[3 * k] * x + Ki[3 * k + 1] * y + Ki[3 * k + 2];
}

// m normalised and negated to face the ray (-ray / |ray| when m is 0 or perpendicular to it), rounded to float.
__device__ __forceinline__ void st_face(double (&m)[3], const double (&ray)[3], float *n)
{
  const double len = sqrt(m[0] * m[0] + m[1] * m[1] + m[2] * m[2]);
  double d = 0.0;
  if (len > 0.0) {
    for (int k = 0; k < 3; k++) m[k] /= len;
    d = m[0] * ray[0] + m[1] * ray[1] + m[2] * ray[2];
  }
  if (d == 0.0) {
    const double rl = sqrt(ray[0] * ray[0] + ray[1] * ray[1] + ray[2] * ray[2]);
    for (int k = 0; k < 3; k++) m[k] = -ray[k] / rl;
  } else if (d > 0.0) {
    for (int k = 0; k < 3; k++) m[k] = -m[k];
  }
  for (int k = 0; k < 3; k++) n[k] = (float)m[k];
}

// The job of thread t of a grid whose jobs start at the threads jobs[].*start (ascending).
__device__ __forceinline__ int st_find(const StJob *__restrict__ jobs, int n, long long StJob::*start, long long t)
{
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].*start <= t) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// The random hypothesis of draws s0 .. s0 + 3.
__device__ __forceinline__ Hyp st_random(const PmParams &P, const StJob &J, int x, int y, int it, int s0,
                                         const double (&ray)[3])
{
  Hyp h;
  const double lo = 1.0 / (double)J.dmax, hi = 1.0 / (double)J.dmin;
  h.z = (float)(1.0 / (lo + st_draw(P.seed, J, x, y, it, s0) * (hi - lo)));
  double m[3];
  for (int k = 0; k < 3; k++) m[k] = 2.0 * st_draw(P.seed, J, x, y, it, s0 + 1 + k) - 1.0;
  st_face(m, ray, h.n);
  return h;
}

// One view's cost of the float homography H at pixel (x, y), or -1 when the view is invalid.
__device__ __forceinline__ float st_view_cost(const StImage &R, const StImage &S, const float (&H)[9], int x, int y, int radius,
                              int step)
{
  const float *ri = R.img;
  const float fx = (float)x, fy = (float)y;
  float q2 = fmaf(H[6], fx, fmaf(H[7], fy, H[8]));
  if (!(q2 > 0.0f)) return -1.0f;
  const float uc = fmaf(H[0], fx, fmaf(H[1], fy, H[2])) / q2, vc = fmaf(H[3], fx, fmaf(H[4], fy, H[5])) / q2;
  if (!(uc >= 0.0f && uc <= (float)(S.w - 1) && vc >= 0.0f && vc <= (float)(S.h - 1))) return -1.0f;
  const float r00 = __ldg(ri + (size_t)y * R.pitch + x);
  const float s00 = st_bilinear(S.img, S.w, S.h, S.pitch, uc, vc);
  float sd = 0.0f, se = 0.0f, sdd = 0.0f, see = 0.0f, sde = 0.0f;
  for (int j = -radius; j <= radius; j += step) {
    const int yy = min(max(y + j, 0), R.h - 1);
    const float fyj = (float)(y + j);
    const float *row = ri + (size_t)yy * R.pitch;
    for (int i = -radius; i <= radius; i += step) {
      const float fxi = (float)(x + i);
      const float w = fmaf(H[6], fxi, fmaf(H[7], fyj, H[8]));
      if (!(w > 0.0f)) return -1.0f;
      const float u = fmaf(H[0], fxi, fmaf(H[1], fyj, H[2])) / w, v = fmaf(H[3], fxi, fmaf(H[4], fyj, H[5])) / w;
      const float d = __ldg(row + min(max(x + i, 0), R.w - 1)) - r00;
      const float e = st_bilinear(S.img, S.w, S.h, S.pitch, u, v) - s00;
      sd += d;
      se += e;
      sdd = fmaf(d, d, sdd);
      see = fmaf(e, e, see);
      sde = fmaf(d, e, sde);
    }
  }
  const int side = 2 * radius / step + 1;
  const float N = (float)(side * side);
  const float md = sd / N, me = se / N;
  const float vd = sdd / N - md * md, ve = see / N - me * me;
  if (!(vd >= ST_VAR_FLOOR) || !(ve >= ST_VAR_FLOOR)) return -1.0f;
  const float c = 1.0f - (sde / N - md * me) / sqrtf(vd * ve);
  return fminf(fmaxf(c, 0.0f), 2.0f);
}

// The aggregated cost of h at (x, y); *invalid counts the invalid views.  Not inlined: a half-step calls it for twelve
// candidates.
__device__ __noinline__ float st_cost(const PmParams &P, const StJob &J, const StImage &R, int x, int y, const Hyp &h,
                         const double (&ray)[3], int *invalid)
{
  float best[ST_MAX_SOURCES];
  const double nr = (double)h.n[0] * ray[0] + (double)h.n[1] * ray[1] + (double)h.n[2] * ray[2];
  const double den = (double)h.z * nr;
  double m[3];
  for (int k = 0; k < 3; k++)
    m[k] = (J.Kinv[k] * h.n[0] + J.Kinv[3 + k] * h.n[1] + J.Kinv[6 + k] * h.n[2]) / den;
  int kept = 0;
  for (int s = 0; s < J.numSources; s++) {
    const StSrc &src = P.srcs[J.src0 + s];
    float H[9];
    for (int a = 0; a < 3; a++)
      for (int k = 0; k < 3; k++) H[3 * a + k] = (float)((double)src.A[3 * a + k] + (double)src.b[a] * m[k]);
    float c = st_view_cost(R, P.images[src.image], H, x, y, P.radius, P.step);
    if (c < 0.0f) { c = 2.0f; (*invalid)++; }
    // insertion into the ascending list of the topK smallest
    int k;
    if (kept < P.topK) k = kept++;
    else if (c < best[P.topK - 1]) k = P.topK - 1;
    else continue;
    while (k > 0 && best[k - 1] > c) { best[k] = best[k - 1]; k--; }
    best[k] = c;
  }
  float sum = 0.0f;
  for (int k = 0; k < P.topK; k++) sum += best[k];
  return sum / (float)P.topK;
}

// The geometric error of the point X (ref camera frame, on the ray of pixel (x, y) of R) in source S, the header's rule
// in float64: forward into S, the prior depth at the nearest pixel, back from the continuous (u, v) into R.  gmax when
// a depth is not positive, q is off S, S has no prior or the prior is not finite or <= 0; *capped when g is gmax.
__device__ __forceinline__ float st_geom_error(const StGeo &G, const StImage &S, const StImage &R, const double (&X)[3],
                                               int x, int y, double gmax, bool *capped)
{
  double e = gmax, Y[3];
  for (int k = 0; k < 3; k++) Y[k] = G.R[3 * k] * X[0] + G.R[3 * k + 1] * X[1] + G.R[3 * k + 2] * X[2] + G.t[k];
  if (G.depth && Y[2] > 0.0) {
    const double u = (S.K[0] * Y[0] + S.K[1] * Y[1] + S.K[2] * Y[2]) / Y[2];
    const double v = (S.K[4] * Y[1] + S.K[5] * Y[2]) / Y[2];
    const double qx = floor(u + 0.5), qy = floor(v + 0.5);
    if (qx >= 0.0 && qx < G.w && qy >= 0.0 && qy < G.h) {
      const double zs = __ldg(G.depth + (size_t)qy * G.w + (size_t)qx);
      if (isfinite(zs) && zs > 0.0) {
        double c[3], Z[3];
        for (int k = 0; k < 3; k++) c[k] = zs * (S.Kinv[3 * k] * u + S.Kinv[3 * k + 1] * v + S.Kinv[3 * k + 2]) - G.t[k];
        for (int k = 0; k < 3; k++) Z[k] = G.R[k] * c[0] + G.R[3 + k] * c[1] + G.R[6 + k] * c[2];
        if (Z[2] > 0.0) {
          const double ex = (R.K[0] * Z[0] + R.K[1] * Z[1] + R.K[2] * Z[2]) / Z[2] - x;
          const double ey = (R.K[4] * Z[1] + R.K[5] * Z[2]) / Z[2] - y;
          e = fmin(hypot(ex, ey), gmax);
        }
      }
    }
  }
  *capped = !(e < gmax);
  return (float)e;
}

// The combined cost of h at (x, y): every view costs fmaf(lambda, g, c_photo), c_photo 2 for an invalid view;
// *invalid counts the invalid views and *capped the valid ones whose g is gmax.  The steps are st_cost's, written out
// again so that st_cost, and with it the photometric kernels, keep their instructions.  Not inlined, as st_cost.
__device__ __noinline__ float st_cost_geom(const PmParams &P, const PmGeom &G, const StJob &J, const StImage &R, int x,
                                           int y, const Hyp &h, const double (&ray)[3], int *invalid, int *capped)
{
  float best[ST_MAX_SOURCES];
  const double nr = (double)h.n[0] * ray[0] + (double)h.n[1] * ray[1] + (double)h.n[2] * ray[2];
  const double den = (double)h.z * nr;
  double m[3], X[3];
  for (int k = 0; k < 3; k++)
    m[k] = (J.Kinv[k] * h.n[0] + J.Kinv[3 + k] * h.n[1] + J.Kinv[6 + k] * h.n[2]) / den;
  for (int k = 0; k < 3; k++) X[k] = (double)h.z * ray[k];
  int kept = 0;
  for (int s = 0; s < J.numSources; s++) {
    const StSrc &src = P.srcs[J.src0 + s];
    const StImage &S = P.images[src.image];
    float H[9];
    for (int a = 0; a < 3; a++)
      for (int k = 0; k < 3; k++) H[3 * a + k] = (float)((double)src.A[3 * a + k] + (double)src.b[a] * m[k]);
    float c = st_view_cost(R, S, H, x, y, P.radius, P.step);
    bool cap;
    const float g = st_geom_error(G.geo[J.src0 + s], S, R, X, x, y, G.gmax, &cap);
    if (c < 0.0f) { c = 2.0f; (*invalid)++; }
    else if (cap) (*capped)++;
    c = fmaf(G.lambda, g, c);
    // insertion into the ascending list of the topK smallest
    int k;
    if (kept < P.topK) k = kept++;
    else if (c < best[P.topK - 1]) k = P.topK - 1;
    else continue;
    while (k > 0 && best[k - 1] > c) { best[k] = best[k - 1]; k--; }
    best[k] = c;
  }
  float sum = 0.0f;
  for (int k = 0; k < P.topK; k++) sum += best[k];
  return sum / (float)P.topK;
}

// The cost of the pass: photometric, or combined with the geometric term.
template <bool GEOM>
__device__ __forceinline__ float st_eval(const PmParams &P, const PmGeom &G, const StJob &J, const StImage &R, int x,
                                         int y, const Hyp &h, const double (&ray)[3], int *invalid, int *capped)
{
  if constexpr (GEOM) return st_cost_geom(P, G, J, R, x, y, h, ray, invalid, capped);
  else return st_cost(P, J, R, x, y, h, ray, invalid);
}

// The warp's lanes of one job add their count to that job's counter k.
__device__ __forceinline__ void st_count(StCounts *counts, int job, int k, unsigned int n)
{
  const unsigned int peers = __match_any_sync(0xffffffffu, job);
  const unsigned int total = __reduce_add_sync(peers, n);
  if (job >= 0 && total && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&counts[job].v[k], (unsigned long long)total);
}

// The ref's prior (z, n) at pixel pix when the header's start rule takes it: z in [depthMin, depthMax], n finite,
// facing the ray and of length 1 within 1e-3.
__device__ __forceinline__ bool st_prior(const StPrior &Pr, const StJob &J, int pix, const double (&ray)[3], Hyp &h)
{
  h.z = Pr.depth[pix];
  for (int k = 0; k < 3; k++) h.n[k] = Pr.normal[3 * (size_t)pix + k];
  if (!(h.z >= J.dmin && h.z <= J.dmax) || !isfinite(h.n[0]) || !isfinite(h.n[1]) || !isfinite(h.n[2])) return false;
  const double d = (double)h.n[0] * ray[0] + (double)h.n[1] * ray[1] + (double)h.n[2] * ray[2];
  const double len = sqrt((double)h.n[0] * h.n[0] + (double)h.n[1] * h.n[1] + (double)h.n[2] * h.n[2]);
  return d < 0.0 && fabs(len - 1.0) <= 1e-3;
}

// Iteration 0.  Photometric: every pixel takes the draws of slot 0.  Geometric: the ref's prior where the start rule
// takes it, else the draws of iteration 32, slot 0.
template <bool GEOM>
__device__ __forceinline__ void pm_start(PmParams P, long long total, PmGeom G)
{
  const long long t = (long long)blockIdx.x * ST_THREADS + threadIdx.x;
  int job = -1, invalid = 0, capped = 0, drawn = 0;
  if (t < total) {
    job = st_find(P.jobs, P.numJobs, &StJob::all0, t);
    const StJob &J = P.jobs[job];
    const int pix = (int)(t - J.all0), x = pix % J.w, y = pix / J.w;
    double ray[3];
    st_ray(J.Kinv, x, y, ray);
    Hyp h;
    if constexpr (GEOM) {
      if (!st_prior(G.priors[job], J, pix, ray, h)) {
        h = st_random(P, J, x, y, ST_GEOM_IT0, 0, ray);
        drawn = 1;
      }
    } else {
      h = st_random(P, J, x, y, 0, 0, ray);
    }
    const float c = st_eval<GEOM>(P, G, J, P.images[J.ref], x, y, h, ray, &invalid, &capped);
    J.depth[pix] = h.z;
    for (int k = 0; k < 3; k++) J.normal[3 * (size_t)pix + k] = h.n[k];
    J.cost[pix] = c;
  }
  st_count(P.counts, job, 1, (unsigned int)invalid);
  if constexpr (GEOM) {
    st_count(G.counts, job, 0, (unsigned int)capped);
    st_count(G.counts, job, 1, (unsigned int)drawn);
  }
}

// One half-step.  The geometric pass keeps rho = 2^-k and draws at counter iteration 32 + k.
template <bool GEOM>
__device__ __forceinline__ void pm_half(PmParams P, long long total, PmGeom G)
{
  const long long t = (long long)blockIdx.x * ST_THREADS + threadIdx.x;
  int job = -1, invalid = 0, capped = 0;
  if (t < total) {
    job = st_find(P.jobs, P.numJobs, &StJob::half0, t);
    const StJob &J = P.jobs[job];
    const int half = (J.w + 1) >> 1, k = (int)(t - J.half0);
    const int y = k / half, x = 2 * (k % half) + ((y + P.colour) & 1);
    if (x < J.w) {
      const StImage &R = P.images[J.ref];
      const int pix = y * J.w + x;
      const int it = GEOM ? ST_GEOM_IT0 + P.iteration : P.iteration;   // the draws' counter iteration
      double ray[3];
      st_ray(J.Kinv, x, y, ray);
      Hyp cur;
      cur.z = J.depth[pix];
      for (int c = 0; c < 3; c++) cur.n[c] = J.normal[3 * (size_t)pix + c];
      Hyp best = cur;
      float bestCost = J.cost[pix];
      auto consider = [&](const Hyp &h) {
        const float c = st_eval<GEOM>(P, G, J, R, x, y, h, ray, &invalid, &capped);
        if (c < bestCost) { bestCost = c; best = h; }
      };
      // 1. propagation
#pragma unroll 1
      for (int q = 0; q < 8; q++) {   // (-1, 0), (1, 0), (0, -1), (0, 1), then the same at distance 5
        const int dist = q < 4 ? 1 : 5, side = (q & 1) ? dist : -dist;
        const int xq = x + ((q & 2) ? 0 : side), yq = y + ((q & 2) ? side : 0);
        if (xq < 0 || xq >= J.w || yq < 0 || yq >= J.h) continue;
        const int pq = yq * J.w + xq;
        Hyp h;
        for (int c = 0; c < 3; c++) h.n[c] = J.normal[3 * (size_t)pq + c];
        double rq[3];
        st_ray(J.Kinv, xq, yq, rq);
        const double zq = J.depth[pq];
        const double d = h.n[0] * ray[0] + h.n[1] * ray[1] + h.n[2] * ray[2];
        if (!(d < 0.0)) continue;
        const double num = zq * ((double)h.n[0] * rq[0] + (double)h.n[1] * rq[1] + (double)h.n[2] * rq[2]);
        h.z = (float)(num / d);
        if (!(h.z >= J.dmin && h.z <= J.dmax)) continue;
        consider(h);
      }
      // 2-4. perturbations
      const double rho = ldexp(1.0, -P.iteration);
      const double lo = 1.0 / (double)J.dmax, hi = 1.0 / (double)J.dmin;
      auto moved_depth = [&](int slot) {
        const double u = st_draw(P.seed, J, x, y, it, slot);
        const double inv = fmin(fmax(1.0 / (double)cur.z + rho * (2.0 * u - 1.0) * (hi - lo), lo), hi);
        return (float)(1.0 / inv);
      };
      auto moved_normal = [&](int slot, float *n) {
        double m[3];
        for (int c = 0; c < 3; c++)
          m[c] = (double)cur.n[c] + rho * (2.0 * st_draw(P.seed, J, x, y, it, slot + c) - 1.0);
        st_face(m, ray, n);
      };
      Hyp h = cur;
      h.z = moved_depth(0);
      consider(h);
      h = cur;
      moved_normal(1, h.n);
      consider(h);
      h.z = moved_depth(4);
      moved_normal(5, h.n);
      consider(h);
      // 5. a fresh random hypothesis
      consider(st_random(P, J, x, y, it, 8, ray));
      J.depth[pix] = best.z;
      for (int c = 0; c < 3; c++) J.normal[3 * (size_t)pix + c] = best.n[c];
      J.cost[pix] = bestCost;
    }
  }
  st_count(P.counts, job, 1, (unsigned int)invalid);
  if constexpr (GEOM) st_count(G.counts, job, 0, (unsigned int)capped);
}

__global__ void __launch_bounds__(ST_THREADS) pm_start_kernel(PmParams P, long long total)
{
  pm_start<false>(P, total, PmGeom{});
}
__global__ void __launch_bounds__(ST_THREADS) pm_half_kernel(PmParams P, long long total)
{
  pm_half<false>(P, total, PmGeom{});
}
__global__ void __launch_bounds__(ST_THREADS) pm_geom_start_kernel(PmParams P, long long total, PmGeom G)
{
  pm_start<true>(P, total, G);
}
__global__ void __launch_bounds__(ST_THREADS) pm_geom_half_kernel(PmParams P, long long total, PmGeom G)
{
  pm_half<true>(P, total, G);
}

__global__ void __launch_bounds__(ST_THREADS) pm_final_kernel(PmParams P, long long total)
{
  const long long t = (long long)blockIdx.x * ST_THREADS + threadIdx.x;
  int job = -1;
  unsigned int bad = 0;
  if (t < total) {
    job = st_find(P.jobs, P.numJobs, &StJob::all0, t);
    const StJob &J = P.jobs[job];
    bad = !(J.cost[t - J.all0] < 2.0f);
  }
  st_count(P.counts, job, 2, bad);
}

// ---- fusion ---------------------------------------------------------------------------------------------------------

struct FuParams {
  const StImage *images;
  const StJob *jobs;       // ascending ref
  const StSrc *srcs;
  int numJobs;
  float maxCost;
  int minConsistent;
  double maxReproj2, maxDepthError, minNormalDot;
  unsigned int *masks, *ctaCounts, *total;
  int rows;
  float *xyz, *normal, *intensity;
  int2 *source;
  int maxPoints;
};

__device__ __forceinline__ void fu_backproject(const StImage &I, double z, double x, double y, double (&X)[3])
{
  double c[3];
  for (int k = 0; k < 3; k++) c[k] = z * (I.Kinv[3 * k] * x + I.Kinv[3 * k + 1] * y + I.Kinv[3 * k + 2]) - I.t[k];
  for (int k = 0; k < 3; k++) X[k] = I.R[k] * c[0] + I.R[3 + k] * c[1] + I.R[6 + k] * c[2];
}

__device__ __forceinline__ void fu_world_normal(const StImage &I, const float *n, double (&w)[3])
{
  for (int k = 0; k < 3; k++) w[k] = I.R[k] * n[0] + I.R[3 + k] * n[1] + I.R[6 + k] * n[2];
}

// Row -> job (ascending ref), its pixel, and the keep rule; with emit the point's sums are formed too.
struct FuPoint {
  double X[3], n[3], inten;
  int views;
};

__device__ bool fu_pixel(const FuParams &P, int row, int &job, int &pix, FuPoint *pt)
{
  job = st_find(P.jobs, P.numJobs, &StJob::all0, row);
  const StJob &J = P.jobs[job];
  pix = row - (int)J.all0;
  if (!(J.cost[pix] <= P.maxCost)) return false;
  const StImage &A = P.images[J.ref];
  const int x = pix % J.w, y = pix / J.w;
  double X[3], n[3];
  fu_backproject(A, J.depth[pix], x, y, X);
  fu_world_normal(A, J.normal + 3 * (size_t)pix, n);
  if (pt) {
    for (int k = 0; k < 3; k++) { pt->X[k] = X[k]; pt->n[k] = n[k]; }
    pt->inten = A.img[(size_t)y * A.pitch + x];
  }
  int good = 0;
  for (int s = 0; s < J.numSources; s++) {
    const int b = P.srcs[J.src0 + s].image;
    const StImage &B = P.images[b];
    if (B.job < 0) continue;
    double Y[3];
    for (int k = 0; k < 3; k++) Y[k] = B.R[3 * k] * X[0] + B.R[3 * k + 1] * X[1] + B.R[3 * k + 2] * X[2] + B.t[k];
    if (!(Y[2] > 0.0)) continue;
    const double u = (B.K[0] * Y[0] + B.K[1] * Y[1] + B.K[2] * Y[2]) / Y[2];
    const double v = (B.K[4] * Y[1] + B.K[5] * Y[2]) / Y[2];
    const double qx = floor(u + 0.5), qy = floor(v + 0.5);
    if (!(qx >= 0.0 && qx < B.w && qy >= 0.0 && qy < B.h)) continue;
    const StJob &JB = P.jobs[B.job];
    const int pq = (int)qy * B.w + (int)qx;
    if (!(JB.cost[pq] <= P.maxCost)) continue;
    const double zb = JB.depth[pq];
    if (!(fabs(zb - Y[2]) <= P.maxDepthError * Y[2])) continue;
    double nb[3];
    fu_world_normal(B, JB.normal + 3 * (size_t)pq, nb);
    if (!(n[0] * nb[0] + n[1] * nb[1] + n[2] * nb[2] >= P.minNormalDot)) continue;
    double Xq[3], Z[3];
    fu_backproject(B, zb, qx, qy, Xq);
    for (int k = 0; k < 3; k++) Z[k] = A.R[3 * k] * Xq[0] + A.R[3 * k + 1] * Xq[1] + A.R[3 * k + 2] * Xq[2] + A.t[k];
    if (!(Z[2] > 0.0)) continue;
    const double ex = (A.K[0] * Z[0] + A.K[1] * Z[1] + A.K[2] * Z[2]) / Z[2] - x;
    const double ey = (A.K[4] * Z[1] + A.K[5] * Z[2]) / Z[2] - y;
    if (!(ex * ex + ey * ey <= P.maxReproj2)) continue;
    if (b < J.ref) return false;
    good++;
    if (pt) {
      for (int k = 0; k < 3; k++) { pt->X[k] += Xq[k]; pt->n[k] += nb[k]; }
      pt->inten += B.img[(size_t)qy * B.pitch + (size_t)qx];
    }
  }
  if (pt) pt->views = good + 1;
  return good >= P.minConsistent;
}

__global__ void __launch_bounds__(LIST_ROWS) fuse_flags_kernel(FuParams P)
{
  const int row = blockIdx.x * LIST_ROWS + threadIdx.x;
  int job, pix;
  const bool keep = row < P.rows && fu_pixel(P, row, job, pix, nullptr);
  list_flag(keep, row, P.rows, P.masks, P.ctaCounts, blockIdx.x);
}

__global__ void __launch_bounds__(LIST_ROWS) fuse_write_kernel(FuParams P)
{
  bool bit;
  const unsigned int at = list_position(P.masks, P.ctaCounts, P.rows, blockIdx.x, &bit, P.total);
  const int row = blockIdx.x * LIST_ROWS + threadIdx.x;
  if (!bit || (int)at >= P.maxPoints) return;
  FuPoint pt;
  int job, pix;
  fu_pixel(P, row, job, pix, &pt);
  const double inv = 1.0 / pt.views;
  const double nl = sqrt(pt.n[0] * pt.n[0] + pt.n[1] * pt.n[1] + pt.n[2] * pt.n[2]);
  for (int k = 0; k < 3; k++) {
    P.xyz[3 * (size_t)at + k] = (float)(pt.X[k] * inv);
    P.normal[3 * (size_t)at + k] = (float)(pt.n[k] / nl);
  }
  P.intensity[at] = (float)(pt.inten * inv);
  P.source[at] = make_int2(P.jobs[job].ref, pix);
}

}  // namespace

// ---- host -----------------------------------------------------------------------------------------------------------

int undistort_images_enqueue(DeviceCtx &c, const cs_image *images, int numImages, const double *Ks,
                             const double *dists, float *const *out, const unsigned long long **outside)
{
  Layout L(256);
  const size_t oTab = L.take(sizeof(UdImage) * numImages), oCnt = L.take(8 * (size_t)numImages);
  int r;
  if ((r = c.stereo.grow(L.bytes)) < 0 || (r = c.h_stereo.grow(L.bytes)) < 0) return r;
  UdImage *t = reinterpret_cast<UdImage *>(c.h_stereo.as<char>() + oTab);
  int gw = 1, gh = 1;
  for (int a = 0; a < numImages; a++) {
    UdImage &m = t[a];
    m.img = images[a].d_img;
    m.out = out[a];
    m.w = images[a].width; m.h = images[a].height; m.pitch = images[a].pitch;
    for (int k = 0; k < 9; k++) m.K[k] = Ks[9 * (size_t)a + k];
    m.k1 = dists ? dists[2 * (size_t)a] : 0.0;
    m.k2 = dists ? dists[2 * (size_t)a + 1] : 0.0;
    gw = std::max(gw, idivup(m.w, 32));
    gh = std::max(gh, idivup(m.h, 8));
  }
  char *d = c.stereo.as<char>();
  unsigned long long *cnt = reinterpret_cast<unsigned long long *>(d + oCnt);
  CS_CUDA(cudaMemcpyAsync(d + oTab, t, sizeof(UdImage) * numImages, cudaMemcpyHostToDevice, c.stream));
  CS_CUDA(cudaMemsetAsync(cnt, 0, 8 * (size_t)numImages, c.stream));
  undistort_images_kernel<<<dim3(gw, gh, std::min(numImages, 65535)), 256, 0, c.stream>>>(
      reinterpret_cast<const UdImage *>(d + oTab), numImages, cnt);
  count_launch();
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaMemcpyAsync(c.h_stereo.as<char>() + oCnt, cnt, 8 * (size_t)numImages, cudaMemcpyDeviceToHost,
                          c.stream));
  *outside = reinterpret_cast<const unsigned long long *>(c.h_stereo.as<char>() + oCnt);
  return 0;
}

namespace {

void inv3(const double *K, double *Ki)
{
  // upper-triangular K with K[8] = 1
  Ki[0] = 1.0 / K[0];
  Ki[1] = -K[1] / (K[0] * K[4]);
  Ki[2] = (K[1] * K[5] - K[2] * K[4]) / (K[0] * K[4]);
  Ki[3] = 0.0;
  Ki[4] = 1.0 / K[4];
  Ki[5] = -K[5] / K[4];
  Ki[6] = Ki[7] = 0.0;
  Ki[8] = 1.0;
}

// The tables of a call, built in c.h_stereo and uploaded to c.stereo: images, jobs (in input order, or sorted by ref
// for fusion), sources, and with priors the geometric table per source and the prior per job; then the job counters
// (a second set with priors); then, for fusion and on the device only, the point list's scratch.
struct StTables {
  StImage *images;
  StJob *jobs;
  StSrc *srcs;
  StGeo *geo;
  StPrior *priors;
  StCounts *counts, *gcounts;
  const StCounts *h_counts;   // the counters' pinned copy (both sets)
  unsigned int *masks, *ctaCounts, *total;
  long long allPixels, halfPixels;
};

int st_tables(DeviceCtx &c, const cs_image *images, int numImages, const double *Ks, const double *Rs,
              const double *ts, const cs_stereo_job *jobs, int numJobs, bool fusion, const cs_depth_prior *priors,
              StTables &T)
{
  std::vector<int> order(numJobs);
  for (int p = 0; p < numJobs; p++) order[p] = p;
  if (fusion) std::sort(order.begin(), order.end(), [&](int a, int b) { return jobs[a].ref < jobs[b].ref; });
  int S = 0;
  long long all = 0, half = 0;
  for (int p = 0; p < numJobs; p++) {
    S += jobs[p].numSources;
    const cs_image &I = images[jobs[p].ref];
    all += (long long)I.width * I.height;
    half += (long long)((I.width + 1) / 2) * I.height;
  }
  const int rows = (int)std::min<long long>(all, INT32_MAX);
  Layout L(256);
  const size_t oIm = L.take(sizeof(StImage) * numImages), oJob = L.take(sizeof(StJob) * numJobs),
               oSrc = L.take(sizeof(StSrc) * std::max(S, 1));
  const size_t oGeo = priors ? L.take(sizeof(StGeo) * std::max(S, 1)) : 0;
  const size_t oPri = priors ? L.take(sizeof(StPrior) * numJobs) : 0, tables = L.bytes;
  const size_t oCnt = L.take(sizeof(StCounts) * numJobs * (priors ? 2 : 1)), hostBytes = L.bytes;
  const size_t oMask = fusion ? L.take(4 * (size_t)list_words(rows)) : 0;
  const size_t oCta = fusion ? L.take(4 * (size_t)list_ctas(rows)) : 0, oTot = fusion ? L.take(4) : 0;
  int r;
  if ((r = c.stereo.grow(L.bytes)) < 0 || (r = c.h_stereo.grow(hostBytes)) < 0) return r;
  char *h = c.h_stereo.as<char>(), *d = c.stereo.as<char>();
  StImage *im = reinterpret_cast<StImage *>(h + oIm);
  StJob *jb = reinterpret_cast<StJob *>(h + oJob);
  StSrc *sr = reinterpret_cast<StSrc *>(h + oSrc);
  StGeo *ge = reinterpret_cast<StGeo *>(h + oGeo);
  StPrior *pr = reinterpret_cast<StPrior *>(h + oPri);
  for (int a = 0; a < numImages; a++) {
    StImage &m = im[a];
    m.img = images[a].d_img;
    m.w = images[a].width; m.h = images[a].height; m.pitch = images[a].pitch;
    m.job = -1;
    for (int k = 0; k < 9; k++) { m.K[k] = Ks[9 * (size_t)a + k]; m.R[k] = Rs[9 * (size_t)a + k]; }
    for (int k = 0; k < 3; k++) m.t[k] = ts[3 * (size_t)a + k];
    inv3(m.K, m.Kinv);
  }
  int s0 = 0;
  all = half = 0;
  for (int q = 0; q < numJobs; q++) {
    const cs_stereo_job &J = jobs[order[q]];
    StJob &j = jb[q];
    const StImage &Rf = im[J.ref];
    im[J.ref].job = q;
    j.ref = J.ref; j.w = Rf.w; j.h = Rf.h;
    j.src0 = s0; j.numSources = J.numSources;
    j.dmin = J.depthMin; j.dmax = J.depthMax;
    for (int k = 0; k < 9; k++) j.Kinv[k] = Rf.Kinv[k];
    j.depth = J.d_depth; j.normal = J.d_normal; j.cost = J.d_cost;
    j.all0 = all; j.half0 = half;
    if (priors) pr[q] = {priors[J.ref].d_depth, priors[J.ref].d_normal};
    all += (long long)j.w * j.h;
    half += (long long)((j.w + 1) / 2) * j.h;
    for (int s = 0; s < J.numSources; s++) {
      const StImage &Sm = im[J.sources[s]];
      StSrc &e = sr[s0 + s];
      e.image = J.sources[s];
      // R_sr = R_s R_r^T, t_sr = t_s - R_sr t_r; A = K_s R_sr Kinv_r, b = K_s t_sr
      double Rsr[9], tsr[3], KR[9];
      for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) {
          double v = 0.0;
          for (int k = 0; k < 3; k++) v += Sm.R[3 * a + k] * Rf.R[3 * b + k];
          Rsr[3 * a + b] = v;
        }
      for (int a = 0; a < 3; a++)
        tsr[a] = Sm.t[a] - (Rsr[3 * a] * Rf.t[0] + Rsr[3 * a + 1] * Rf.t[1] + Rsr[3 * a + 2] * Rf.t[2]);
      for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++)
          KR[3 * a + b] = Sm.K[3 * a] * Rsr[b] + Sm.K[3 * a + 1] * Rsr[3 + b] + Sm.K[3 * a + 2] * Rsr[6 + b];
      for (int a = 0; a < 3; a++) {
        for (int b = 0; b < 3; b++)
          e.A[3 * a + b] = (float)(KR[3 * a] * Rf.Kinv[b] + KR[3 * a + 1] * Rf.Kinv[3 + b] + KR[3 * a + 2] * Rf.Kinv[6 + b]);
        e.b[a] = (float)(Sm.K[3 * a] * tsr[0] + Sm.K[3 * a + 1] * tsr[1] + Sm.K[3 * a + 2] * tsr[2]);
      }
      if (priors) {
        StGeo &g = ge[s0 + s];
        for (int k = 0; k < 9; k++) g.R[k] = Rsr[k];
        for (int k = 0; k < 3; k++) g.t[k] = tsr[k];
        g.depth = priors[e.image].d_depth;
        g.w = Sm.w; g.h = Sm.h;
      }
    }
    s0 += J.numSources;
  }
  CS_CUDA(cudaMemcpyAsync(d, h, tables, cudaMemcpyHostToDevice, c.stream));
  T.images = reinterpret_cast<StImage *>(d + oIm);
  T.jobs = reinterpret_cast<StJob *>(d + oJob);
  T.srcs = reinterpret_cast<StSrc *>(d + oSrc);
  T.geo = priors ? reinterpret_cast<StGeo *>(d + oGeo) : nullptr;
  T.priors = priors ? reinterpret_cast<StPrior *>(d + oPri) : nullptr;
  T.counts = reinterpret_cast<StCounts *>(d + oCnt);
  T.gcounts = priors ? T.counts + numJobs : nullptr;
  T.h_counts = reinterpret_cast<const StCounts *>(h + oCnt);
  T.masks = fusion ? reinterpret_cast<unsigned int *>(d + oMask) : nullptr;
  T.ctaCounts = fusion ? reinterpret_cast<unsigned int *>(d + oCta) : nullptr;
  T.total = fusion ? reinterpret_cast<unsigned int *>(d + oTot) : nullptr;
  T.allPixels = all;
  T.halfPixels = half;
  return 0;
}

}  // namespace

namespace {

// The launches of a PatchMatch call (start, the half-steps, the final count) and the counters' copy back; with G the
// geometric kernels.
int pm_launch(DeviceCtx &c, const StTables &T, PmParams P, int numIterations, const PmGeom *G,
              const unsigned long long **counts)
{
  const int sets = G ? 2 : 1;
  CS_CUDA(cudaMemsetAsync(T.counts, 0, sizeof(StCounts) * P.numJobs * sets, c.stream));
  const unsigned int gAll = (unsigned int)((T.allPixels + ST_THREADS - 1) / ST_THREADS);
  const unsigned int gHalf = (unsigned int)((T.halfPixels + ST_THREADS - 1) / ST_THREADS);
  if (G) pm_geom_start_kernel<<<gAll, ST_THREADS, 0, c.stream>>>(P, T.allPixels, *G);
  else pm_start_kernel<<<gAll, ST_THREADS, 0, c.stream>>>(P, T.allPixels);
  count_launch();
  CS_CUDA(cudaGetLastError());
  for (int it = 1; it <= numIterations; it++)
    for (int colour = 0; colour < 2; colour++) {
      P.iteration = it;
      P.colour = colour;
      if (G) pm_geom_half_kernel<<<gHalf, ST_THREADS, 0, c.stream>>>(P, T.halfPixels, *G);
      else pm_half_kernel<<<gHalf, ST_THREADS, 0, c.stream>>>(P, T.halfPixels);
      count_launch();
      CS_CUDA(cudaGetLastError());
    }
  pm_final_kernel<<<gAll, ST_THREADS, 0, c.stream>>>(P, T.allPixels);
  count_launch();
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaMemcpyAsync(const_cast<StCounts *>(T.h_counts), T.counts, sizeof(StCounts) * P.numJobs * sets,
                          cudaMemcpyDeviceToHost, c.stream));
  *counts = T.h_counts->v;
  return 0;
}

}  // namespace

int patch_match_enqueue(DeviceCtx &c, const cs_image *images, int numImages, const double *Ks, const double *Rs,
                        const double *ts, const cs_stereo_job *jobs, int numJobs, int radius, int step,
                        int numIterations, int topK, unsigned long long seed, const unsigned long long **counts)
{
  StTables T;
  int r;
  if ((r = st_tables(c, images, numImages, Ks, Rs, ts, jobs, numJobs, false, nullptr, T)) < 0) return r;
  const PmParams P{T.images, T.jobs, T.srcs, T.counts, numJobs, radius, step, topK, seed, 0, 0};
  return pm_launch(c, T, P, numIterations, nullptr, counts);
}

int patch_match_geometric_enqueue(DeviceCtx &c, const cs_image *images, int numImages, const double *Ks,
                                  const double *Rs, const double *ts, const cs_depth_prior *priors,
                                  const cs_stereo_job *jobs, int numJobs, int radius, int step, int numIterations,
                                  int topK, double geomWeight, double geomMaxError, unsigned long long seed,
                                  const unsigned long long **counts)
{
  StTables T;
  int r;
  if ((r = st_tables(c, images, numImages, Ks, Rs, ts, jobs, numJobs, false, priors, T)) < 0) return r;
  const PmParams P{T.images, T.jobs, T.srcs, T.counts, numJobs, radius, step, topK, seed, 0, 0};
  const PmGeom G{T.geo, T.priors, T.gcounts, (float)geomWeight, geomMaxError};
  return pm_launch(c, T, P, numIterations, &G, counts);
}

int fuse_enqueue(DeviceCtx &c, const cs_image *images, int numImages, const double *Ks, const double *Rs,
                 const double *ts, const cs_stereo_job *jobs, int numJobs, float maxCost, int minConsistent,
                 double maxReprojError, double maxDepthError, double maxNormalErrorDeg, float *xyz, float *normal,
                 float *intensity, int *source, int maxPoints, unsigned int **total)
{
  StTables T;
  int r;
  if ((r = st_tables(c, images, numImages, Ks, Rs, ts, jobs, numJobs, true, nullptr, T)) < 0) return r;
  FuParams P;
  P.images = T.images; P.jobs = T.jobs; P.srcs = T.srcs; P.numJobs = numJobs;
  P.maxCost = maxCost; P.minConsistent = minConsistent;
  P.maxReproj2 = maxReprojError * maxReprojError;
  P.maxDepthError = maxDepthError;
  P.minNormalDot = cos(maxNormalErrorDeg * (CUDART_PI / 180.0));
  P.masks = T.masks; P.ctaCounts = T.ctaCounts; P.total = T.total;
  P.rows = (int)T.allPixels;
  P.xyz = xyz; P.normal = normal; P.intensity = intensity; P.source = reinterpret_cast<int2 *>(source);
  P.maxPoints = maxPoints;
  const int ctas = list_ctas(P.rows);
  fuse_flags_kernel<<<ctas, LIST_ROWS, 0, c.stream>>>(P);
  count_launch();
  CS_CUDA(cudaGetLastError());
  fuse_write_kernel<<<ctas, LIST_ROWS, 0, c.stream>>>(P);
  count_launch();
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaMemcpyAsync(c.h_counters, T.total, 4, cudaMemcpyDeviceToHost, c.stream));
  *total = c.h_counters;
  return 0;
}

}  // namespace cs
