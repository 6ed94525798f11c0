// refine.cu -- photometric mesh refinement (cs_mesh_refine) after Vu, Labatut, Pons & Keriven (PAMI 2012): gradient
// descent of every free vertex on the windowed NCC reprojection error of ordered image pairs through the mesh, plus a
// thin-plate term, with a halving line search.  Every rule is stated in cudasift_b200.h at cs_mesh_refine;
// tests/refine_oracle.py restates them in float64.
//
// Per evaluation: the depth buffers of every paired image (cs_texture_mesh's rule 2, restated here so texture.o keeps
// its instructions), then per pair four image passes over the ref image (map, score with the tile partials of e, the
// pair total, the image gradient) and a warp per face that gathers s phi_k over the face's visible pixels in the
// photo kernel's lane and butterfly order; then the thin plate and the vertex gradient with their totals.  The vertex
// sums run over the sorted directed edge keys and the corners sorted by vertex, so every sum has a fixed order.
//
// Determinism: no floating-point atomics; integer atomics only where the result does not depend on their order (the
// depth keys, the flags, the counts).  The totals use coop.cuh's three-level order.  This unit is compiled with
// -fmad=false so that every float64 product and sum is rounded once, in the order written, as the oracle computes it.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include <cub/cub.cuh>

#include "common.cuh"
#include "coop.cuh"
#include "trimesh.cuh"

namespace cs {

namespace {

constexpr unsigned long long EMPTY = ~0ull;

// One image a pair names: its pixels, size, camera and depth buffer.
struct RefCam {
  const float *img;
  int W, H, pitch;
  double K[9], R[9], t[3], C[3];
  unsigned long long *buf;
};

// The device words of a call, copied back after the input check, the setup and each evaluation.
struct RefineResult {
  unsigned int bad;
  unsigned int free;                          // free vertices
  unsigned long long scored;                  // scored pixels of the evaluation, over all pairs
  unsigned long long P0;                      // scored pixels of the first evaluation
  double edgeLen;                             // the sum of the distinct undirected edge lengths
  double es;                                  // the total of |U|^2 over the free vertices
  double g2;                                  // the total of |G|^2 over the free vertices
};

struct RefineParams {
  RefineResult *res;
  int V, T, numCams;
  const float *vin;                           // the vertices of the evaluation (setup: the input)
  const int *tin;
  const RefCam *cams;
  unsigned long long *dkey, *dkeyS;           // [6T] directed edge keys and sorted
  int *ckey, *ckeyS, *cval, *cvalS;           // [3T] corner vertices and corners, sorted by vertex
  int *head, *hidx;                           // [6T + 1] run heads and their exclusive scan
  int *nb;                                    // [distinct directed edges] the neighbour of each
  int *flag;                                  // [V] bit 0: used by a face, bit 1: on an edge not held by two faces
  int2 *nrange, *crange;                      // [V] ranges of the neighbour list and of the sorted corners
  double *acc;                                // [3T] the corner sums of s phi_k
  double *U;                                  // [V][3] the thin-plate vectors
  double *part, *group;                       // tile and group partials
  double *pairTot;                            // [numPairs] each pair's total of e
  // the pair being processed
  int ci, cj, rho;
  double depthTol;
  double *J, *c, *terms;                      // [pixels], [pixels] (c, then s), [pixels][4] {A, B, Cc, D}
  unsigned char *mapped, *scored;             // [pixels]
};

// Y = R X + t, (u, v) = (K Y)_{0,1} / Y_z (rule 2 of cs_texture_mesh)
__device__ __forceinline__ void project(const RefCam &c, D3 X, double &u, double &v, double &z)
{
  const double y0 = ((c.R[0] * X.x + c.R[1] * X.y) + c.R[2] * X.z) + c.t[0];
  const double y1 = ((c.R[3] * X.x + c.R[4] * X.y) + c.R[5] * X.z) + c.t[1];
  const double y2 = ((c.R[6] * X.x + c.R[7] * X.y) + c.R[8] * X.z) + c.t[2];
  u = ((c.K[0] * y0 + c.K[1] * y1) + c.K[2] * y2) / y2;
  v = ((c.K[3] * y0 + c.K[4] * y1) + c.K[5] * y2) / y2;
  z = y2;
}

// A face in one image: its vertex ids, float64 corners, their projections, the sign of the doubled area and its
// clipped box; ok when rule 2 rasterises it.
struct FaceView {
  int id[3];
  D3 P[3];
  double u[3], v[3], z[3];
  EdgeFns ef;
  int x0, y0, x1, y1;
  bool ok;
};

__device__ __forceinline__ void face_view(const RefineParams &p, const RefCam &c, int f, FaceView &fv)
{
  bool front = true;
  for (int k = 0; k < 3; k++) {
    fv.id[k] = p.tin[3 * (size_t)f + k];
    fv.P[k] = vertex_of(p.vin, fv.id[k]);
    project(c, fv.P[k], fv.u[k], fv.v[k], fv.z[k]);
    front = front && fv.z[k] > 0.0;
  }
  fv.ok = false;
  if (!front) return;
  const double A = (fv.u[1] - fv.u[0]) * (fv.v[2] - fv.v[0]) - (fv.v[1] - fv.v[0]) * (fv.u[2] - fv.u[0]);
  if (!(A != 0.0) || !isfinite(A)) return;
  const double xlo = fmax(0.0, ceil(fmin(fmin(fv.u[0], fv.u[1]), fv.u[2]))),
               xhi = fmin(c.W - 1.0, floor(fmax(fmax(fv.u[0], fv.u[1]), fv.u[2])));
  const double ylo = fmax(0.0, ceil(fmin(fmin(fv.v[0], fv.v[1]), fv.v[2]))),
               yhi = fmin(c.H - 1.0, floor(fmax(fmax(fv.v[0], fv.v[1]), fv.v[2])));
  if (!(xlo <= xhi && ylo <= yhi)) return;
  fv.x0 = (int)xlo;
  fv.x1 = (int)xhi;
  fv.y0 = (int)ylo;
  fv.y1 = (int)yhi;
  edge_fns_of(fv.id, fv.u, fv.v, A > 0.0 ? 1.0 : -1.0, fv.ef);
  fv.ok = true;
}

// rule 3's perspective-correct weights phi_k at pixel (x, y) of a face that covers it
__device__ __forceinline__ void weights_at(const FaceView &fv, int x, int y, double (&phi)[3])
{
  double w[3];
  for (int k = 0; k < 3; k++) w[k] = edge_fn(fv.ef, fv.u, fv.v, k, (double)x, (double)y);
  const double S = (w[0] + w[1]) + w[2];
  const double t0 = (w[1] / S) / fv.z[0], t1 = (w[2] / S) / fv.z[1], t2 = (w[0] / S) / fv.z[2];
  const double sum = (t0 + t1) + t2;
  phi[0] = t0 / sum;
  phi[1] = t1 / sum;
  phi[2] = t2 / sum;
}

__device__ __forceinline__ double pixel_at(const RefCam &c, int x, int y)
{
  return (double)c.img[(size_t)y * c.pitch + x];
}

// ---- setup (rule 1) -----------------------------------------------------------------------------------------------
// corner c = 3t + k, edge a -> b: directed keys (a, b) at 2c and (b, a) at 2c + 1; the corner's vertex keyed for the
// corner sort
__global__ void __launch_bounds__(MT) refine_keys_kernel(RefineParams p)
{
  for (int c = blockIdx.x * MT + threadIdx.x; c < 3 * p.T; c += gridDim.x * MT) {
    const int t = c / 3, k = c - 3 * t;
    const unsigned int a = p.tin[c], b = p.tin[3 * t + (k + 1) % 3];
    p.dkey[2 * (size_t)c] = ((unsigned long long)a << 32) | b;
    p.dkey[2 * (size_t)c + 1] = ((unsigned long long)b << 32) | a;
    p.ckey[c] = (int)a;
    p.cval[c] = c;
  }
}

// run heads of the sorted directed keys, the flags of the run's first vertex, and the corner ranges
__global__ void __launch_bounds__(MT) refine_runs_kernel(RefineParams p)
{
  const int n = 6 * p.T;
  for (int i = blockIdx.x * MT + threadIdx.x; i <= n; i += gridDim.x * MT) {
    if (i == n) { p.head[n] = 0; continue; }
    const unsigned long long k = p.dkeyS[i];
    const bool h = i == 0 || p.dkeyS[i - 1] != k;
    p.head[i] = h;
    if (h) {
      int m = 1;
      while (i + m < n && p.dkeyS[i + m] == k) m++;
      atomicOr(&p.flag[(int)(k >> 32)], m == 2 ? 1 : 3);
    }
    if (i < 3 * p.T) {
      const int a = p.ckeyS[i];
      if (i == 0 || p.ckeyS[i - 1] != a) p.crange[a].x = i;
      if (i == 3 * p.T - 1 || p.ckeyS[i + 1] != a) p.crange[a].y = i + 1;
    }
  }
}

// The neighbour list and its ranges from the scanned heads, the free count, and the tile partials of the lengths of
// the distinct undirected edges (heads with a < b), over the sorted positions.
__global__ void __launch_bounds__(MT) refine_compact_kernel(RefineParams p)
{
  unsigned int nfree = 0;
  for (int v = blockIdx.x * MT + threadIdx.x; v < p.V; v += gridDim.x * MT) nfree += p.flag[v] == 1;
  if (nfree) atomicAdd(&p.res->free, nfree);
  const int n = 6 * p.T;
  co_tree_tiles<1, MT>(n, p.part, [&](int i, double *s) {
    const unsigned long long k = p.dkeyS[i];
    const int a = (int)(k >> 32), b = (int)(unsigned int)k;
    if (i == 0 || (int)(p.dkeyS[i - 1] >> 32) != a) p.nrange[a].x = p.hidx[i];
    if (i == n - 1 || (int)(p.dkeyS[i + 1] >> 32) != a) p.nrange[a].y = p.hidx[i] + p.head[i];
    if (!p.head[i]) return;
    p.nb[p.hidx[i]] = b;
    if (a < b) {
      const D3 d = sub3(vertex_of(p.vin, b), vertex_of(p.vin, a));
      s[0] += sqrt(dot3(d, d));
    }
  });
}

// one CTA: the total of n items' tile partials into *out
__global__ void __launch_bounds__(MT) refine_total_kernel(RefineParams p, int n, double *out)
{
  double tot[1];
  co_tree_groups<1, MT>(n, p.part, p.group);
  co_tree_total<1, MT>(n, p.group, tot);
  if (threadIdx.x == 0) *out = tot[0];
}

// ---- depth buffers (rule 2) ---------------------------------------------------------------------------------------
// cs_texture_mesh's raster: one thread per (paired image, face), 64-bit atomicMin of (float(depth) bits << 32) | face
__global__ void __launch_bounds__(MT) refine_raster_kernel(RefineParams p)
{
  const long long n = (long long)p.numCams * p.T;
  for (long long i = blockIdx.x * (long long)MT + threadIdx.x; i < n; i += (long long)gridDim.x * MT) {
    const int g = (int)(i / p.T), f = (int)(i % p.T);
    const RefCam &c = p.cams[g];
    FaceView fv;
    face_view(p, c, f, fv);
    if (!fv.ok) continue;
    for (int y = fv.y0; y <= fv.y1; y++)
      for (int x = fv.x0; x <= fv.x1; x++) {
        double w[3];
        bool in = true;
        for (int k = 0; k < 3 && in; k++) {
          w[k] = edge_fn(fv.ef, fv.u, fv.v, k, (double)x, (double)y);
          in = w[k] >= 0.0;
        }
        if (!in) continue;
        const double W = (w[0] + w[1]) + w[2];
        if (!(W > 0.0)) continue;
        const double iz = ((w[1] / fv.z[0] + w[2] / fv.z[1]) + w[0] / fv.z[2]) / W;
        const float d = __double2float_rn(1.0 / iz);
        atomicMin(c.buf + (size_t)y * c.W + x, ((unsigned long long)__float_as_uint(d) << 32) | (unsigned int)f);
      }
  }
}

// ---- per pair (rules 3 to 6) --------------------------------------------------------------------------------------
// rule 3 at every pixel of image i: J and the chain factor c of the mapped pixels
__global__ void __launch_bounds__(MT) refine_map_kernel(RefineParams p)
{
  const RefCam &I = p.cams[p.ci], &Jc = p.cams[p.cj];
  const int n = I.W * I.H;
  for (int q = blockIdx.x * MT + threadIdx.x; q < n; q += gridDim.x * MT) {
    unsigned char m = 0;
    const unsigned long long key = I.buf[q];
    if (key != EMPTY) {
      const int f = (int)(unsigned int)key, y = q / I.W, x = q - y * I.W;
      FaceView fv;
      face_view(p, I, f, fv);
      double phi[3];
      weights_at(fv, x, y, phi);
      const D3 X = {(phi[0] * fv.P[0].x + phi[1] * fv.P[1].x) + phi[2] * fv.P[2].x,
                    (phi[0] * fv.P[0].y + phi[1] * fv.P[1].y) + phi[2] * fv.P[2].y,
                    (phi[0] * fv.P[0].z + phi[1] * fv.P[1].z) + phi[2] * fv.P[2].z};
      const D3 r = sub3(X, {I.C[0], I.C[1], I.C[2]});
      const double nr = dot3(normal3(fv.P[0], fv.P[1], fv.P[2]), r);
      double u, v, z;
      project(Jc, X, u, v, z);
      bool ok = z > 0.0 && u >= 0.0 && u <= Jc.W - 1.0 && v >= 0.0 && v <= Jc.H - 1.0 && nr != 0.0;
      if (ok) {
        const unsigned long long kj = Jc.buf[(size_t)(int)floor(v + 0.5) * Jc.W + (int)floor(u + 0.5)];
        ok = kj == EMPTY || (unsigned int)kj == (unsigned int)f ||
             z <= (double)__uint_as_float((unsigned int)(kj >> 32)) * (1.0 + p.depthTol);
      }
      if (ok) {
        const int x0 = min((int)floor(u), Jc.W - 2), y0 = min((int)floor(v), Jc.H - 2);
        const double fx = u - x0, fy = v - y0;
        const double I00 = pixel_at(Jc, x0, y0), I10 = pixel_at(Jc, x0 + 1, y0), I01 = pixel_at(Jc, x0, y0 + 1),
                     I11 = pixel_at(Jc, x0 + 1, y0 + 1);
        const double a = I00 + fx * (I10 - I00), b = I01 + fx * (I11 - I01);
        const double gu = (I10 - I00) + fy * ((I11 - I01) - (I10 - I00)), gv = b - a;
        const double d0 = (Jc.R[0] * r.x + Jc.R[1] * r.y) + Jc.R[2] * r.z;
        const double d1 = (Jc.R[3] * r.x + Jc.R[4] * r.y) + Jc.R[5] * r.z;
        const double d2 = (Jc.R[6] * r.x + Jc.R[7] * r.y) + Jc.R[8] * r.z;
        const double au = (((Jc.K[0] * d0 + Jc.K[1] * d1) + Jc.K[2] * d2) - u * d2) / z;
        const double av = (((Jc.K[3] * d0 + Jc.K[4] * d1) + Jc.K[5] * d2) - v * d2) / z;
        p.J[q] = a + fy * (b - a);
        p.c[q] = (gu * au + gv * av) / nr;
        m = 1;
      }
    }
    p.mapped[q] = m;
  }
}

// rule 4: the scored pixels, their terms A, B, Cc, D (rule 5) and the tile partials of e; counts the scored pixels
__global__ void __launch_bounds__(MT) refine_score_kernel(RefineParams p)
{
  const RefCam &I = p.cams[p.ci];
  const int W = I.W, H = I.H, rho = p.rho;
  const double n = (double)((2 * rho + 1) * (2 * rho + 1));
  unsigned int count = 0;
  co_tree_tiles<1, MT>(W * H, p.part, [&](int q, double *s) {
    const int y = q / W, x = q - y * W;
    bool ok = x >= rho && x < W - rho && y >= rho && y < H - rho;
    for (int dy = -rho; dy <= rho && ok; dy++)
      for (int dx = -rho; dx <= rho && ok; dx++) ok = p.mapped[q + dy * W + dx] != 0;
    p.scored[q] = ok;
    if (!ok) return;
    double sI = 0.0, sJ = 0.0, sII = 0.0, sJJ = 0.0, sIJ = 0.0;
    for (int dy = -rho; dy <= rho; dy++)
      for (int dx = -rho; dx <= rho; dx++) {
        const double a = pixel_at(I, x + dx, y + dy), b = p.J[q + dy * W + dx];
        sI = sI + a;
        sJ = sJ + b;
        sII = sII + a * a;
        sJJ = sJJ + b * b;
        sIJ = sIJ + a * b;
      }
    const double mI = sI / n, mJ = sJ / n;
    const double rI = sII / n - mI * mI, rJ = sJJ / n - mJ * mJ;
    const double vI = rI < 1.0 ? 1.0 : rI, vJ = rJ < 1.0 ? 1.0 : rJ;
    const double qq = sqrt(vI * vJ);
    const double ncc = (sIJ / n - mI * mJ) / qq;
    const double A = 1.0 / qq, Cc = rJ < 1.0 ? 0.0 : ncc / vJ;
    double *t = p.terms + 4 * (size_t)q;
    t[0] = A;
    t[1] = mI * A;
    t[2] = Cc;
    t[3] = Cc * mJ;
    s[0] += 1.0 - ncc;
    count++;
  });
  if (count) atomicAdd(&p.res->scored, (unsigned long long)count);
}

// rule 5: s(y) = dE/dJ(y) c(y) at every mapped pixel, into c
__global__ void __launch_bounds__(MT) refine_back_kernel(RefineParams p)
{
  const RefCam &I = p.cams[p.ci];
  const int W = I.W, H = I.H, rho = p.rho;
  const double n = (double)((2 * rho + 1) * (2 * rho + 1));
  for (int q = blockIdx.x * MT + threadIdx.x; q < W * H; q += gridDim.x * MT) {
    if (!p.mapped[q]) continue;
    const int y = q / W, x = q - y * W;
    double SA = 0.0, SB = 0.0, SC = 0.0, SD = 0.0;
    for (int dy = -rho; dy <= rho; dy++)
      for (int dx = -rho; dx <= rho; dx++) {
        const int xx = x + dx, yy = y + dy;
        if (xx < 0 || xx >= W || yy < 0 || yy >= H) continue;
        const int o = yy * W + xx;
        if (!p.scored[o]) continue;
        const double *t = p.terms + 4 * (size_t)o;
        SA = SA + t[0];
        SB = SB + t[1];
        SC = SC + t[2];
        SD = SD + t[3];
      }
    const double g = ((pixel_at(I, x, y) * SA - SB) - p.J[q] * SC) + SD;
    p.c[q] = (-g / n) * p.c[q];
  }
}

// rule 6: a warp per face, s phi_k over its mapped visible pixels in image i (lane-strided, xor butterfly), added to
// the corner sums
__global__ void __launch_bounds__(MT) refine_face_kernel(RefineParams p)
{
  const RefCam &I = p.cams[p.ci];
  const int lane = threadIdx.x & 31;
  for (int f = blockIdx.x * (MT / 32) + (threadIdx.x >> 5); f < p.T; f += gridDim.x * (MT / 32)) {
    double S[3] = {0.0, 0.0, 0.0};
    FaceView fv;
    face_view(p, I, f, fv);
    if (fv.ok) {
      const int bw = fv.x1 - fv.x0 + 1, N = bw * (fv.y1 - fv.y0 + 1);
      for (int i = lane; i < N; i += 32) {
        const int dy = i / bw, x = fv.x0 + (i - dy * bw), y = fv.y0 + dy;
        const int q = y * I.W + x;
        if ((unsigned int)I.buf[q] != (unsigned int)f || !p.mapped[q]) continue;
        double phi[3];
        weights_at(fv, x, y, phi);
        const double s = p.c[q];
        S[0] = S[0] + s * phi[0];
        S[1] = S[1] + s * phi[1];
        S[2] = S[2] + s * phi[2];
      }
    }
    for (int o = 16; o > 0; o >>= 1)
      for (int k = 0; k < 3; k++) S[k] = S[k] + __shfl_xor_sync(~0u, S[k], o);
    if (lane == 0)
      for (int k = 0; k < 3; k++) p.acc[3 * (size_t)f + k] = p.acc[3 * (size_t)f + k] + S[k];
  }
}

// ---- per vertex (rules 6 to 8) ------------------------------------------------------------------------------------
// rule 7: U of every free vertex and the tile partials of |U|^2
__global__ void __launch_bounds__(MT) refine_thin_kernel(RefineParams p)
{
  co_tree_tiles<1, MT>(p.V, p.part, [&](int v, double *s) {
    double *U = p.U + 3 * (size_t)v;
    if (p.flag[v] != 1) return;
    const int2 r = p.nrange[v];
    D3 a = {0.0, 0.0, 0.0};
    for (int j = r.x; j < r.y; j++) {
      const D3 w = vertex_of(p.vin, p.nb[j]);
      a = {a.x + w.x, a.y + w.y, a.z + w.z};
    }
    const double deg = (double)(r.y - r.x);
    const D3 P = vertex_of(p.vin, v);
    U[0] = a.x / deg - P.x;
    U[1] = a.y / deg - P.y;
    U[2] = a.z / deg - P.z;
    s[0] += (U[0] * U[0] + U[1] * U[1]) + U[2] * U[2];
  });
}

// rules 6 and 7: G of every free vertex (0 for the fixed ones) and the tile partials of |G|^2
__global__ void __launch_bounds__(MT) refine_grad_kernel(RefineParams p, const unsigned long long *P0, double ks,
                                                         double smoothness, double *G)
{
  const double p0 = (double)*P0;
  co_tree_tiles<1, MT>(p.V, p.part, [&](int v, double *s) {
    double *g = G + 3 * (size_t)v;
    g[0] = g[1] = g[2] = 0.0;
    if (p.flag[v] != 1) return;
    const int2 cr = p.crange[v];
    D3 a = {0.0, 0.0, 0.0};
    for (int j = cr.x; j < cr.y; j++) {
      const int c = p.cvalS[j], f = c / 3;
      const D3 nf = normal3(vertex_of(p.vin, p.tin[3 * f]), vertex_of(p.vin, p.tin[3 * f + 1]),
                            vertex_of(p.vin, p.tin[3 * f + 2]));
      const double w = p.acc[c];
      a = {a.x + w * nf.x, a.y + w * nf.y, a.z + w * nf.z};
    }
    const double *U = p.U + 3 * (size_t)v;
    D3 b = {-U[0], -U[1], -U[2]};
    const int2 r = p.nrange[v];
    for (int j = r.x; j < r.y; j++) {
      const int w = p.nb[j];
      if (p.flag[w] != 1) continue;
      const double dw = (double)(p.nrange[w].y - p.nrange[w].x);
      const double *Uw = p.U + 3 * (size_t)w;
      b = {b.x + Uw[0] / dw, b.y + Uw[1] / dw, b.z + Uw[2] / dw};
    }
    g[0] = a.x / p0 + smoothness * (ks * b.x);
    g[1] = a.y / p0 + smoothness * (ks * b.y);
    g[2] = a.z / p0 + smoothness * (ks * b.z);
    s[0] += (g[0] * g[0] + g[1] * g[1]) + g[2] * g[2];
  });
}

// rule 8: the candidate, float(V + Delta) for the free vertices, the others copied
__global__ void __launch_bounds__(MT) refine_step_kernel(RefineParams p, const double *G, double scale, double cap,
                                                         float *out)
{
  for (int v = blockIdx.x * MT + threadIdx.x; v < p.V; v += gridDim.x * MT) {
    const D3 P = vertex_of(p.vin, v);
    float *o = out + 3 * (size_t)v;
    if (p.flag[v] != 1) {
      o[0] = p.vin[3 * (size_t)v];
      o[1] = p.vin[3 * (size_t)v + 1];
      o[2] = p.vin[3 * (size_t)v + 2];
      continue;
    }
    const double *g = G + 3 * (size_t)v;
    double d[3] = {-(scale * g[0]), -(scale * g[1]), -(scale * g[2])};
    const double len = sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]);
    if (len > cap) {
      const double f = cap / len;
      for (int k = 0; k < 3; k++) d[k] = d[k] * f;
    }
    o[0] = __double2float_rn(P.x + d[0]);
    o[1] = __double2float_rn(P.y + d[1]);
    o[2] = __double2float_rn(P.z + d[2]);
  }
}

// CTAs of a three-level tile pass over n items: one per tile of CO_TREE_TILE, at least 1, at most 8192
int tiles_of(long long n) { return (int)std::max(1ll, std::min((n + CO_TREE_TILE - 1) / CO_TREE_TILE, 8192ll)); }

}  // namespace

int refine_run(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
               const float *vin, int V, const int *tin, int T, const int *pairs, int numPairs, int windowRadius,
               double smoothness, double step, int maxIterations, double depthTol, float *outVertices,
               cudaStream_t st, void *h_res, double *info, long long *stats)
{
  const size_t C3 = 3 * (size_t)T, C6 = 6 * (size_t)T;
  // the paired images in ascending order, and each pair's two slots
  std::vector<int> slotOf(numImages, -1), used;
  for (int q = 0; q < numPairs; q++)
    for (int e = 0; e < 2; e++) slotOf[pairs[2 * q + e]] = 0;
  for (int a = 0; a < numImages; a++)
    if (slotOf[a] == 0) {
      slotOf[a] = (int)used.size();
      used.push_back(a);
    }
  const int M = (int)used.size();
  size_t bufPix = 0, refPix = 1;
  for (int a : used) bufPix += (size_t)images[a].width * images[a].height;
  for (int q = 0; q < numPairs; q++) {
    const cs_image &I = images[pairs[2 * q]];
    refPix = std::max(refPix, (size_t)I.width * I.height);
  }
  size_t tb[3] = {};
  CS_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb[0], (unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                         (int)C6, 0, 64, st));
  CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb[1], (int *)nullptr, (int *)nullptr, (int *)nullptr,
                                          (int *)nullptr, (int)C3, 0, 32, st));
  CS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb[2], (int *)nullptr, (int *)nullptr, (int)C6 + 1, st));
  size_t tempBytes = std::max(tb[0], std::max(tb[1], tb[2]));
  const long long most = std::max((long long)std::max(C6, (size_t)V), (long long)refPix);
  const int tiles = (int)((most + CO_TREE_TILE - 1) / CO_TREE_TILE), groups = (tiles + MT - 1) / MT;

  Layout L(256);
  const size_t resAt = L.take(sizeof(RefineResult)), camAt = L.take((size_t)std::max(M, 1) * sizeof(RefCam));
  const size_t dkAt = L.take(C6 * 8), dkSAt = L.take(C6 * 8), ckAt = L.take(C3 * 4), ckSAt = L.take(C3 * 4),
               cvAt = L.take(C3 * 4), cvSAt = L.take(C3 * 4), headAt = L.take((C6 + 1) * 4),
               hidxAt = L.take((C6 + 1) * 4), nbAt = L.take(C6 * 4), accAt = L.take(C3 * 8);
  const size_t flagAt = L.take((size_t)V * 4), nrAt = L.take((size_t)V * 8), crAt = L.take((size_t)V * 8),
               uAt = L.take((size_t)V * 24), gAt = L.take((size_t)V * 24), g2At = L.take((size_t)V * 24),
               candAt = L.take((size_t)V * 12);
  const size_t partAt = L.take((size_t)tiles * 8), groupAt = L.take((size_t)groups * 8),
               pairAt = L.take((size_t)std::max(numPairs, 1) * 8);
  const size_t bufAt = L.take(bufPix * 8);
  const size_t jAt = L.take(refPix * 8), cAt = L.take(refPix * 8), termAt = L.take(refPix * 32),
               mapAt = L.take(refPix), scAt = L.take(refPix);
  const size_t tempAt = L.take(tempBytes);
  char *base = nullptr;
  CS_CUDA(cudaMallocAsync((void **)&base, L.bytes, st));
  auto at = [&](size_t off) { return base + off; };

  std::vector<RefCam> cams(std::max(M, 1));
  size_t off = 0;
  unsigned long long *buf = reinterpret_cast<unsigned long long *>(at(bufAt));
  for (int s = 0; s < M; s++) {
    const int a = used[s];
    RefCam &c = cams[s];
    c.img = images[a].d_img;
    c.W = images[a].width;
    c.H = images[a].height;
    c.pitch = images[a].pitch;
    for (int k = 0; k < 9; k++) c.K[k] = Ks[9 * (size_t)a + k], c.R[k] = Rs[9 * (size_t)a + k];
    for (int k = 0; k < 3; k++) c.t[k] = ts[3 * (size_t)a + k];
    for (int i = 0; i < 3; i++) c.C[i] = -((c.R[i] * c.t[0] + c.R[3 + i] * c.t[1]) + c.R[6 + i] * c.t[2]);
    c.buf = buf + off;
    off += (size_t)c.W * c.H;
  }

  RefineParams p{};
  p.res = reinterpret_cast<RefineResult *>(at(resAt));
  p.V = V;
  p.T = T;
  p.numCams = M;
  p.vin = vin;
  p.tin = tin;
  p.cams = reinterpret_cast<const RefCam *>(at(camAt));
  p.dkey = reinterpret_cast<unsigned long long *>(at(dkAt));
  p.dkeyS = reinterpret_cast<unsigned long long *>(at(dkSAt));
  p.ckey = reinterpret_cast<int *>(at(ckAt));
  p.ckeyS = reinterpret_cast<int *>(at(ckSAt));
  p.cval = reinterpret_cast<int *>(at(cvAt));
  p.cvalS = reinterpret_cast<int *>(at(cvSAt));
  p.head = reinterpret_cast<int *>(at(headAt));
  p.hidx = reinterpret_cast<int *>(at(hidxAt));
  p.nb = reinterpret_cast<int *>(at(nbAt));
  p.flag = reinterpret_cast<int *>(at(flagAt));
  p.nrange = reinterpret_cast<int2 *>(at(nrAt));
  p.crange = reinterpret_cast<int2 *>(at(crAt));
  p.acc = reinterpret_cast<double *>(at(accAt));
  p.U = reinterpret_cast<double *>(at(uAt));
  p.part = reinterpret_cast<double *>(at(partAt));
  p.group = reinterpret_cast<double *>(at(groupAt));
  p.pairTot = reinterpret_cast<double *>(at(pairAt));
  p.rho = windowRadius;
  p.depthTol = depthTol;
  p.J = reinterpret_cast<double *>(at(jAt));
  p.c = reinterpret_cast<double *>(at(cAt));
  p.terms = reinterpret_cast<double *>(at(termAt));
  p.mapped = reinterpret_cast<unsigned char *>(at(mapAt));
  p.scored = reinterpret_cast<unsigned char *>(at(scAt));
  double *Gacc = reinterpret_cast<double *>(at(gAt)), *Gcand = reinterpret_cast<double *>(at(g2At));
  float *cand = reinterpret_cast<float *>(at(candAt));
  void *temp = at(tempAt);
  RefineResult &R = *static_cast<RefineResult *>(h_res);
  cudaEvent_t *tev = match_timing_events();

  int status = 0, evals = 0, accepted = 0, halvings = 0;
  unsigned long long P0 = 0;
  double l0 = 0.0, Ds = 0.0, ks = 0.0, e0[2] = {0.0, 0.0}, eAcc[2] = {0.0, 0.0};
  std::vector<double> pairTot(std::max(numPairs, 1));
  auto readback = [&]() -> int {
    CS_CUDA(cudaMemcpyAsync(h_res, p.res, sizeof(RefineResult), cudaMemcpyDeviceToHost, st));
    CS_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  // one evaluation of E and G at verts: E_photo and E_s into e, the total of |G|^2 into *g2
  auto evaluate = [&](const float *verts, double *G, double (&e)[2], double &g2) -> int {
    int r;
    const bool first = evals == 0;
    p.vin = verts;
    CS_CUDA(cudaMemsetAsync(&p.res->scored, 0, 8, st));
    CS_CUDA(cudaMemsetAsync(p.acc, 0, C3 * 8, st));
    if (bufPix) CS_CUDA(cudaMemsetAsync(buf, 0xff, bufPix * 8, st));
    refine_raster_kernel<<<grid_of((long long)M * T), MT, 0, st>>>(p);
    count_launch();
    CS_CUDA(cudaGetLastError());
    if (tev && first) CS_CUDA(cudaEventRecord(tev[2], st));
    for (int q = 0; q < numPairs; q++) {
      p.ci = slotOf[pairs[2 * q]];
      p.cj = slotOf[pairs[2 * q + 1]];
      const long long n = (long long)cams[p.ci].W * cams[p.ci].H;
      refine_map_kernel<<<grid_of(n), MT, 0, st>>>(p);
      refine_score_kernel<<<tiles_of(n), MT, 0, st>>>(p);
      refine_total_kernel<<<1, MT, 0, st>>>(p, (int)n, p.pairTot + q);
      refine_back_kernel<<<grid_of(n), MT, 0, st>>>(p);
      refine_face_kernel<<<grid_of(32ll * T), MT, 0, st>>>(p);
      count_launch(5);
      CS_CUDA(cudaGetLastError());
    }
    if (tev && first) CS_CUDA(cudaEventRecord(tev[3], st));
    if (first) CS_CUDA(cudaMemcpyAsync(&p.res->P0, &p.res->scored, 8, cudaMemcpyDeviceToDevice, st));
    refine_thin_kernel<<<tiles_of(V), MT, 0, st>>>(p);
    refine_total_kernel<<<1, MT, 0, st>>>(p, V, &p.res->es);
    refine_grad_kernel<<<tiles_of(V), MT, 0, st>>>(p, &p.res->P0, ks, smoothness, G);
    refine_total_kernel<<<1, MT, 0, st>>>(p, V, &p.res->g2);
    count_launch(4);
    CS_CUDA(cudaGetLastError());
    if (tev && first) CS_CUDA(cudaEventRecord(tev[4], st));
    if (numPairs) CS_CUDA(cudaMemcpyAsync(pairTot.data(), p.pairTot, (size_t)numPairs * 8, cudaMemcpyDeviceToHost, st));
    if ((r = readback()) < 0) return r;
    evals++;
    if (first) P0 = R.P0;
    double sum = 0.0;
    for (int q = 0; q < numPairs; q++) sum = sum + pairTot[q];
    e[0] = P0 ? sum / (double)P0 : 0.0;
    e[1] = Ds > 0.0 ? R.es / Ds : 0.0;
    g2 = R.g2;
    return 0;
  };
  auto energy = [&](const double (&e)[2]) { return e[0] + smoothness * e[1]; };
  auto run = [&]() -> int {
    int r;
    if (tev) CS_CUDA(cudaEventRecord(tev[0], st));
    CS_CUDA(cudaMemsetAsync(p.res, 0, sizeof(RefineResult), st));
    mesh_validate_kernel<<<grid_of(T), MT, 0, st>>>(vin, V, tin, T, &p.res->bad);
    count_launch();
    CS_CUDA(cudaGetLastError());
    if ((r = readback()) < 0) return r;
    if (R.bad) {
      status = 2;
      return 0;
    }
    if (M) CS_CUDA(cudaMemcpyAsync(at(camAt), cams.data(), (size_t)M * sizeof(RefCam), cudaMemcpyHostToDevice, st));
    CS_CUDA(cudaMemsetAsync(p.flag, 0, (size_t)V * 4, st));
    CS_CUDA(cudaMemsetAsync(p.nrange, 0, (size_t)V * 8, st));
    CS_CUDA(cudaMemsetAsync(p.crange, 0, (size_t)V * 8, st));
    CS_CUDA(cudaMemsetAsync(p.U, 0, (size_t)V * 24, st));
    refine_keys_kernel<<<grid_of((long long)C3), MT, 0, st>>>(p);
    CS_CUDA(cub::DeviceRadixSort::SortKeys(temp, tempBytes, p.dkey, p.dkeyS, (int)C6, 0, 64, st));
    CS_CUDA(cub::DeviceRadixSort::SortPairs(temp, tempBytes, p.ckey, p.ckeyS, p.cval, p.cvalS, (int)C3, 0, 32, st));
    refine_runs_kernel<<<grid_of((long long)C6 + 1), MT, 0, st>>>(p);
    CS_CUDA(cub::DeviceScan::ExclusiveSum(temp, tempBytes, p.head, p.hidx, (int)C6 + 1, st));
    refine_compact_kernel<<<tiles_of((long long)C6), MT, 0, st>>>(p);
    refine_total_kernel<<<1, MT, 0, st>>>(p, (int)C6, &p.res->edgeLen);
    count_launch(4);
    CS_CUDA(cudaGetLastError());
    int distinct = 0;
    CS_CUDA(cudaMemcpyAsync(&distinct, p.hidx + C6, 4, cudaMemcpyDeviceToHost, st));
    if ((r = readback()) < 0) return r;
    l0 = R.edgeLen / (double)(distinct / 2);
    Ds = (double)R.free * (l0 * l0);
    ks = Ds > 0.0 ? 2.0 / Ds : 0.0;
    if (tev) CS_CUDA(cudaEventRecord(tev[1], st));
    // the accepted vertices live in outVertices
    CS_CUDA(cudaMemcpyAsync(outVertices, vin, (size_t)V * 12, cudaMemcpyDeviceToDevice, st));
    if ((r = evaluate(outVertices, Gacc, e0, R.g2)) < 0) return r;
    eAcc[0] = e0[0];
    eAcc[1] = e0[1];
    if (tev) {
      static const char *const names[4] = {"setup", "raster", "pairs", "vertices"};
      report_stage_times(tev, names, 4, "refine timing faces=%d vertices=%d images=%d pairs=%d", T, V, M, numPairs);
    }
    if (P0 == 0) {
      status = 1;
      return 0;
    }
    double gAcc = R.g2, alpha = step;
    for (;;) {
      const double grms = R.free ? std::sqrt(gAcc / (double)R.free) : 0.0;
      if (grms == 0.0 || alpha < step / 1024.0) { status = 0; break; }
      if (evals - 1 == maxIterations) { status = 3; break; }
      const double al = alpha * l0;
      p.vin = outVertices;
      refine_step_kernel<<<grid_of(V), MT, 0, st>>>(p, Gacc, al / grms, 2.0 * al, cand);
      count_launch();
      CS_CUDA(cudaGetLastError());
      double e[2], g2 = 0.0;
      if ((r = evaluate(cand, Gcand, e, g2)) < 0) return r;
      if (energy(e) < energy(eAcc)) {
        CS_CUDA(cudaMemcpyAsync(outVertices, cand, (size_t)V * 12, cudaMemcpyDeviceToDevice, st));
        std::swap(Gacc, Gcand);
        eAcc[0] = e[0];
        eAcc[1] = e[1];
        gAcc = g2;
        accepted++;
        alpha = step;
        halvings = 0;
      } else {
        alpha = alpha * 0.5;
        halvings++;
      }
    }
    CS_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  const int r = run();
  cudaFreeAsync(base, st);
  if (r < 0) return r;
  const bool out = status != 2;
  if (info) {
    info[0] = out ? e0[0] : 0.0;
    info[1] = out ? e0[1] : 0.0;
    info[2] = out ? eAcc[0] : 0.0;
    info[3] = out ? eAcc[1] : 0.0;
  }
  if (stats) {
    stats[0] = numPairs;
    stats[1] = out ? R.free : 0;
    stats[2] = out ? V - (long long)R.free : 0;
    stats[3] = (long long)P0;
    stats[4] = evals;
    stats[5] = accepted;
    stats[6] = halvings;
    stats[7] = status;
  }
  return status;
}

size_t refine_result_bytes() { return sizeof(RefineResult); }

}  // namespace cs
