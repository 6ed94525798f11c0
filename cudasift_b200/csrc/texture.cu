// texture.cu -- mesh texturing (cs_texture_mesh) after Waechter, Moehrle & Goesele 2014, without seam levelling: the
// face adjacency by a radix sort of undirected edge keys, a depth buffer per image by 64-bit atomicMin of (depth, face)
// keys, one thread per face for the visibility tests and its best candidates, a Jones-Plassmann colouring of the face
// graph, ICM sweeps over the colours, charts by union-find, the shelf packing on the host, and the texel copy.  Every
// rule is stated in cudasift_b200.h at cs_texture_mesh; tests/texture_oracle.py restates them in float64.  The float64
// vectors, the colouring priority s(f), the input check and the launch shape are shared with simplify.cu in
// trimesh.cuh; the union-find is common.cuh's (uf_find, uf_link), shared with tracks.cu.  cs_texture_mesh_photo runs
// the same body with a warp per face in place of the candidate thread (each passing view sampled over the face's
// visible pixels for its Sobel magnitude and mean intensity) and one outlier kernel before the labelling; its rules
// are stated at cs_texture_mesh_photo and restated in tests/texture_photo_oracle.py.  cs_texture_mesh_bp is the photo
// call with min-sum belief propagation between the colouring and the ICM sweeps: a message step per colour, a decode
// and the energy total per sweep, the labelling of lowest energy kept (rule 4b, tests/texture_bp_oracle.py).
//
// Determinism: no floating-point atomics; integer atomics only where the result does not depend on their order (the
// depth keys, counts, union-find links to the lower root, the chart rectangles).  The energy totals use coop.cuh's
// three-level order.  This unit is compiled with -fmad=false so that every float64 product and sum is rounded once, in
// the order written, as the oracle computes it.
#include <climits>
#include <cmath>
#include <cstring>

#include <cub/cub.cuh>

#include "common.cuh"
#include "coop.cuh"
#include "trimesh.cuh"

namespace cs {

long long g_texture_group_bytes = 0;          // cs_set_tuning("texture_group_bytes"); 0: TEXTURE_GROUP_BYTES

namespace {

constexpr int MCAND = 8;                      // candidates a face keeps
constexpr long long TEXTURE_GROUP_BYTES = 1ll << 30;
constexpr unsigned long long EMPTY = ~0ull;

// One image of the call: its pixels, size, camera and, in the group being processed, its depth buffer.
struct TexCam {
  const float *img;
  int W, H, pitch;
  double K[9], R[9], t[3], C[3];
  unsigned long long *buf;
};

// The device words of a call, copied back after each step that decides the next.
struct TextureResult {
  unsigned int bad;
  unsigned int cand;                          // (face, image) pairs that passed every test
  unsigned int unseen;
  unsigned int left;                          // uncoloured faces after a round
  int maxColour;
  unsigned int changed;                       // labels changed in a sweep
  int charts;                                 // exclusive scan of the root flags at T
  double energy;
};

struct TextureParams {
  TextureResult *res;
  int V, T, numImages;
  const float *vin;
  const int *tin;
  const TexCam *cams;
  int g0, gn;                                 // the images of the current group
  unsigned long long *ekey, *ekeyS;           // edge keys [3T] and sorted
  int *eval, *evalS;                          // their corners
  int *nbr;                                   // [3T]: the face across edge k of f, or -1
  double *cq;                                 // [T][MCAND] candidate quality
  int *ca, *cn;                               // [T][MCAND] candidate image, [T] count
  int *label, *colA, *colB, *parent, *flag, *chartIdx;
  double *part, *group;                       // energy tile and group partials
  double lambda, cosLim, depthTol;
  int padding;
  int *craw;                                  // [C][6] {image, xmin, ymin, xmax, ymax, faces}
  const int *ctab;                            // [C][8] the chart table of cs_texture_mesh
  const long long *cstart;                    // [C + 1] first texel of each chart
  int numCharts;
  float *atlas, *uv;
  int *faceView, *faceChart;
  int atlasWidth, rowsWritten;
};

// Y = R X + t, (u, v) = (K Y)_{0,1} / Y_z (rule 2)
__device__ __forceinline__ void project(const TexCam &c, D3 X, double &u, double &v, double &z)
{
  const double y0 = ((c.R[0] * X.x + c.R[1] * X.y) + c.R[2] * X.z) + c.t[0];
  const double y1 = ((c.R[3] * X.x + c.R[4] * X.y) + c.R[5] * X.z) + c.t[1];
  const double y2 = ((c.R[6] * X.x + c.R[7] * X.y) + c.R[8] * X.z) + c.t[2];
  u = ((c.K[0] * y0 + c.K[1] * y1) + c.K[2] * y2) / y2;
  v = ((c.K[3] * y0 + c.K[4] * y1) + c.K[5] * y2) / y2;
  z = y2;
}

// The doubled signed area of a projected face, corners in face order.
__device__ __forceinline__ double area2_of(const double *u, const double *v)
{
  return (u[1] - u[0]) * (v[2] - v[0]) - (v[1] - v[0]) * (u[2] - u[0]);
}

// ---- input and adjacency (rule 1) ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(MT) texture_edges_kernel(TextureParams p)
{
  for (int c = blockIdx.x * MT + threadIdx.x; c < 3 * p.T; c += gridDim.x * MT) {
    p.ekey[c] = edge_key_of(p.tin, c);
    p.eval[c] = c;
    p.nbr[c] = -1;
  }
}

// a run of exactly two equal keys in the sorted list joins its two faces
__global__ void __launch_bounds__(MT) texture_adjacency_kernel(TextureParams p)
{
  const int n = 3 * p.T;
  for (int i = blockIdx.x * MT + threadIdx.x; i + 1 < n; i += gridDim.x * MT) {
    edge_pair_join(p.ekeyS, p.evalS, p.nbr, i, n);
  }
}

// ---- depth buffers (rule 2) ---------------------------------------------------------------------------------------
// One thread per (image of the group, face): every pixel centre of the clipped bounding box that the three oriented
// edge functions cover gets atomicMin of (float(depth) bits << 32) | face.
__global__ void __launch_bounds__(MT) texture_raster_kernel(TextureParams p)
{
  const long long n = (long long)p.gn * p.T;
  for (long long i = blockIdx.x * (long long)MT + threadIdx.x; i < n; i += (long long)gridDim.x * MT) {
    const int g = p.g0 + (int)(i / p.T), f = (int)(i % p.T);
    const TexCam &c = p.cams[g];
    int id[3];
    double u[3], v[3], z[3];
    bool front = true;
    for (int k = 0; k < 3; k++) {
      id[k] = p.tin[3 * (size_t)f + k];
      project(c, vertex_of(p.vin, id[k]), u[k], v[k], z[k]);
      front = front && z[k] > 0.0;
    }
    if (!front) continue;
    const double A = area2_of(u, v);
    if (!(A != 0.0) || !isfinite(A)) continue;
    const double s = A > 0.0 ? 1.0 : -1.0;
    const double xlo = fmax(0.0, ceil(fmin(fmin(u[0], u[1]), u[2]))), xhi = fmin(c.W - 1.0, floor(fmax(fmax(u[0], u[1]), u[2])));
    const double ylo = fmax(0.0, ceil(fmin(fmin(v[0], v[1]), v[2]))), yhi = fmin(c.H - 1.0, floor(fmax(fmax(v[0], v[1]), v[2])));
    if (!(xlo <= xhi && ylo <= yhi)) continue;
    EdgeFns ef;
    edge_fns_of(id, u, v, s, ef);
    for (int y = (int)ylo; y <= (int)yhi; y++)
      for (int x = (int)xlo; x <= (int)xhi; x++) {
        double w[3];
        bool in = true;
        for (int k = 0; k < 3 && in; k++) {
          w[k] = edge_fn(ef, u, v, k, (double)x, (double)y);
          in = w[k] >= 0.0;
        }
        if (!in) continue;
        const double W = (w[0] + w[1]) + w[2];
        if (!(W > 0.0)) continue;
        const double iz = ((w[1] / z[0] + w[2] / z[1]) + w[0] / z[2]) / W;
        const float d = __double2float_rn(1.0 / iz);
        atomicMin(c.buf + (size_t)y * c.W + x, ((unsigned long long)__float_as_uint(d) << 32) | (unsigned int)f);
      }
  }
}

// ---- candidates (rule 3) ------------------------------------------------------------------------------------------
__device__ __forceinline__ bool sees(const TexCam &c, D3 X, int f, double depthTol, double &u, double &v)
{
  double z;
  project(c, X, u, v, z);
  if (!(z > 0.0 && u >= 0.0 && u <= c.W - 1.0 && v >= 0.0 && v <= c.H - 1.0)) return false;
  const int px = (int)floor(u + 0.5), py = (int)floor(v + 0.5);
  const unsigned long long key = c.buf[(size_t)py * c.W + px];
  if (key == EMPTY || (unsigned int)key == (unsigned int)f) return true;
  return z <= (double)__uint_as_float((unsigned int)(key >> 32)) * (1.0 + depthTol);
}

// One thread per face: the images of the group in ascending order, each that passes every test inserted into the
// face's list by (q descending, image ascending), at most MCAND kept.
__global__ void __launch_bounds__(MT) texture_candidate_kernel(TextureParams p)
{
  unsigned int found = 0;
  for (int f = blockIdx.x * MT + threadIdx.x; f < p.T; f += gridDim.x * MT) {
    const D3 p0 = vertex_of(p.vin, p.tin[3 * (size_t)f]), p1 = vertex_of(p.vin, p.tin[3 * (size_t)f + 1]),
             p2 = vertex_of(p.vin, p.tin[3 * (size_t)f + 2]);
    const D3 n = normal3(p0, p1, p2);
    const D3 cen = {((p0.x + p1.x) + p2.x) / 3.0, ((p0.y + p1.y) + p2.y) / 3.0, ((p0.z + p1.z) + p2.z) / 3.0};
    const double ln = sqrt(dot3(n, n));
    double *cq = p.cq + (size_t)f * MCAND;
    int *ca = p.ca + (size_t)f * MCAND;
    int cnt = p.cn[f];
    for (int g = p.g0; g < p.g0 + p.gn; g++) {
      const TexCam &c = p.cams[g];
      const D3 d = sub3({c.C[0], c.C[1], c.C[2]}, cen);
      const double dn = dot3(n, d);
      if (!(dn > 0.0) || !(dn >= p.cosLim * (ln * sqrt(dot3(d, d))))) continue;
      double u[3], v[3], uc, vc;
      if (!sees(c, p0, f, p.depthTol, u[0], v[0]) || !sees(c, p1, f, p.depthTol, u[1], v[1]) ||
          !sees(c, p2, f, p.depthTol, u[2], v[2]) || !sees(c, cen, f, p.depthTol, uc, vc))
        continue;
      const double q = 0.5 * fabs(area2_of(u, v));
      if (!(q > 0.0)) continue;
      found++;
      int r = cnt < MCAND ? cnt : MCAND;
      while (r > 0 && (q > cq[r - 1] || (q == cq[r - 1] && g < ca[r - 1]))) {
        if (r < MCAND) { cq[r] = cq[r - 1]; ca[r] = ca[r - 1]; }
        r--;
      }
      if (r < MCAND) { cq[r] = q; ca[r] = g; }
      if (cnt < MCAND) cnt++;
    }
    p.cn[f] = cnt;
  }
  if (found) atomicAdd(&p.res->cand, found);
}

// ---- candidates of cs_texture_mesh_photo (rules 3a to 3c) ---------------------------------------------------------
// The photo call's device words and settings travel as a second kernel argument, so TextureParams and TextureResult
// keep their layout and the kernels above their instructions.
struct PhotoResult {
  unsigned long long samples;                 // visible pixels summed over the passing pairs
  unsigned long long fallbacks;               // passing pairs with no visible pixel centre
  unsigned int tested, removed, bestRemoved;
};

struct PhotoParams {
  PhotoResult *res;
  double *mu;                                 // [T][MCAND] mean intensity of each kept candidate
  int dataTerm;                               // 0 area, 1 GMI
  double outlierK, minSigma;
};

// pixel (x, y) of c, indices clamped to the image
__device__ __forceinline__ double pixel_at(const TexCam &c, int x, int y)
{
  x = min(max(x, 0), c.W - 1);
  y = min(max(y, 0), c.H - 1);
  return (double)c.img[(size_t)y * c.pitch + x];
}

// the Sobel magnitude at (x, y) over 8, so that a ramp of slope s gives s (rule 3a)
__device__ __forceinline__ double sobel_at(const TexCam &c, int x, int y)
{
  const double gx = ((pixel_at(c, x + 1, y - 1) - pixel_at(c, x - 1, y - 1)) +
                     2.0 * (pixel_at(c, x + 1, y) - pixel_at(c, x - 1, y))) +
                    (pixel_at(c, x + 1, y + 1) - pixel_at(c, x - 1, y + 1));
  const double gy = ((pixel_at(c, x - 1, y + 1) - pixel_at(c, x - 1, y - 1)) +
                     2.0 * (pixel_at(c, x, y + 1) - pixel_at(c, x, y - 1))) +
                    (pixel_at(c, x + 1, y + 1) - pixel_at(c, x + 1, y - 1));
  return sqrt(gx * gx + gy * gy) / 8.0;
}

// A warp per face: lane l runs rule 3's tests for image b + l of the group, a ballot collects the images that pass,
// then the warp samples each of them in ascending order (lane j the box indices j mod 32, the sums combined by the
// xor butterfly) and lane 0 inserts it with its mean intensity, as texture_candidate_kernel does.
__global__ void __launch_bounds__(MT) texture_photo_candidate_kernel(TextureParams p, PhotoParams h)
{
  const int lane = threadIdx.x & 31;
  unsigned int found = 0;
  unsigned long long samples = 0, fallbacks = 0;
  for (int f = blockIdx.x * (MT / 32) + (threadIdx.x >> 5); f < p.T; f += gridDim.x * (MT / 32)) {
    const D3 p0 = vertex_of(p.vin, p.tin[3 * (size_t)f]), p1 = vertex_of(p.vin, p.tin[3 * (size_t)f + 1]),
             p2 = vertex_of(p.vin, p.tin[3 * (size_t)f + 2]);
    const D3 n = normal3(p0, p1, p2);
    const D3 cen = {((p0.x + p1.x) + p2.x) / 3.0, ((p0.y + p1.y) + p2.y) / 3.0, ((p0.z + p1.z) + p2.z) / 3.0};
    const double ln = sqrt(dot3(n, n));
    double *cq = p.cq + (size_t)f * MCAND, *mu = h.mu + (size_t)f * MCAND;
    int *ca = p.ca + (size_t)f * MCAND;
    int cnt = p.cn[f];
    for (int b = p.g0; b < p.g0 + p.gn; b += 32) {
      bool pass = false;
      const int g = b + lane;
      if (g < p.g0 + p.gn) {
        const TexCam &c = p.cams[g];
        const D3 d = sub3({c.C[0], c.C[1], c.C[2]}, cen);
        const double dn = dot3(n, d);
        double u[3], v[3], uc, vc;
        pass = dn > 0.0 && dn >= p.cosLim * (ln * sqrt(dot3(d, d))) && sees(c, p0, f, p.depthTol, u[0], v[0]) &&
               sees(c, p1, f, p.depthTol, u[1], v[1]) && sees(c, p2, f, p.depthTol, u[2], v[2]) &&
               sees(c, cen, f, p.depthTol, uc, vc) && 0.5 * fabs(area2_of(u, v)) > 0.0;
      }
      for (unsigned int m = __ballot_sync(~0u, pass); m; m &= m - 1) {
        const int a = b + __ffs(m) - 1;
        const TexCam &c = p.cams[a];
        double u[3], v[3], z, uc, vc;
        project(c, p0, u[0], v[0], z);
        project(c, p1, u[1], v[1], z);
        project(c, p2, u[2], v[2], z);
        project(c, cen, uc, vc, z);
        const double area = 0.5 * fabs(area2_of(u, v));
        // rule 2's clipped box of f in image a; its samples are the pixels whose key names f
        const double xlo = fmax(0.0, ceil(fmin(fmin(u[0], u[1]), u[2]))), xhi = fmin(c.W - 1.0, floor(fmax(fmax(u[0], u[1]), u[2])));
        const double ylo = fmax(0.0, ceil(fmin(fmin(v[0], v[1]), v[2]))), yhi = fmin(c.H - 1.0, floor(fmax(fmax(v[0], v[1]), v[2])));
        int cntS = 0;
        double sg = 0.0, si = 0.0;
        if (xlo <= xhi && ylo <= yhi) {
          const int x0 = (int)xlo, y0 = (int)ylo, bw = (int)xhi - x0 + 1, N = bw * ((int)yhi - y0 + 1);
          for (int i = lane; i < N; i += 32) {
            const int dy = i / bw, x = x0 + (i - dy * bw), y = y0 + dy;
            if ((unsigned int)c.buf[(size_t)y * c.W + x] != (unsigned int)f) continue;
            cntS++;
            sg = sg + sobel_at(c, x, y);
            si = si + pixel_at(c, x, y);
          }
        }
        for (int o = 16; o > 0; o >>= 1) {
          cntS += __shfl_xor_sync(~0u, cntS, o);
          sg = sg + __shfl_xor_sync(~0u, sg, o);
          si = si + __shfl_xor_sync(~0u, si, o);
        }
        double gm, mean;
        if (cntS > 0) {
          gm = sg / (double)cntS;
          mean = si / (double)cntS;
        } else {
          const int px = (int)floor(uc + 0.5), py = (int)floor(vc + 0.5);
          gm = sobel_at(c, px, py);
          mean = pixel_at(c, px, py);
        }
        const double q = h.dataTerm ? area * (gm + 1.0) : area;
        if (lane == 0) {
          found++;
          samples += (unsigned int)cntS;
          fallbacks += cntS == 0;
          int r = cnt < MCAND ? cnt : MCAND;
          while (r > 0 && (q > cq[r - 1] || (q == cq[r - 1] && a < ca[r - 1]))) {
            if (r < MCAND) { cq[r] = cq[r - 1]; ca[r] = ca[r - 1]; mu[r] = mu[r - 1]; }
            r--;
          }
          if (r < MCAND) { cq[r] = q; ca[r] = a; mu[r] = mean; }
        }
        if (cnt < MCAND) cnt++;
      }
    }
    if (lane == 0) p.cn[f] = cnt;
  }
  if (found) atomicAdd(&p.res->cand, found);
  if (samples) atomicAdd(&h.res->samples, samples);
  if (fallbacks) atomicAdd(&h.res->fallbacks, fallbacks);
}

// the median of s [m], sorted in place: the middle value, or (a + b) * 0.5 of the two middle values for even m
__device__ __forceinline__ double median_of(double *s, int m)
{
  for (int i = 1; i < m; i++)
    for (int j = i; j > 0 && s[j] < s[j - 1]; j--) {
      const double t = s[j];
      s[j] = s[j - 1];
      s[j - 1] = t;
    }
  return m & 1 ? s[m / 2] : (s[m / 2 - 1] + s[m / 2]) * 0.5;
}

// One thread per face (rule 3c): with outlierK > 0 and m >= 3 kept candidates, every candidate whose mean is further
// than outlierK max(1.4826 MAD, minSigma) from the median of the means leaves the list; the survivors keep their order.
__global__ void __launch_bounds__(MT) texture_outlier_kernel(TextureParams p, PhotoParams h)
{
  unsigned int tested = 0, removed = 0, best = 0;
  for (int f = blockIdx.x * MT + threadIdx.x; f < p.T; f += gridDim.x * MT) {
    const int m = p.cn[f];
    if (!(h.outlierK > 0.0) || m < 3) continue;
    double *cq = p.cq + (size_t)f * MCAND, *mu = h.mu + (size_t)f * MCAND;
    int *ca = p.ca + (size_t)f * MCAND;
    double s[MCAND];
    for (int i = 0; i < m; i++) s[i] = mu[i];
    const double med = median_of(s, m);
    for (int i = 0; i < m; i++) s[i] = fabs(mu[i] - med);
    const double lim = h.outlierK * fmax(1.4826 * median_of(s, m), h.minSigma);
    best += fabs(mu[0] - med) > lim;
    int k = 0;
    for (int i = 0; i < m; i++) {
      if (fabs(mu[i] - med) > lim) continue;
      cq[k] = cq[i];
      ca[k] = ca[i];
      mu[k] = mu[i];
      k++;
    }
    tested++;
    removed += m - k;
    p.cn[f] = k;
  }
  if (tested) atomicAdd(&h.res->tested, tested);
  if (removed) atomicAdd(&h.res->removed, removed);
  if (best) atomicAdd(&h.res->bestRemoved, best);
}

// ---- labelling (rule 4) -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MT) texture_label_init_kernel(TextureParams p)
{
  unsigned int unseen = 0;
  for (int f = blockIdx.x * MT + threadIdx.x; f < p.T; f += gridDim.x * MT) {
    const bool seen = p.cn[f] > 0;
    p.label[f] = seen ? p.ca[(size_t)f * MCAND] : -1;
    unseen += !seen;
    p.colA[f] = -1;
    p.parent[f] = f;
  }
  if (unseen) atomicAdd(&p.res->unseen, unseen);
}

// A Jones-Plassmann round: reads colA (the state at its start), writes colB.
__global__ void __launch_bounds__(MT) texture_colour_kernel(TextureParams p)
{
  unsigned int left = 0;
  int top = -1;
  for (int f = blockIdx.x * MT + threadIdx.x; f < p.T; f += gridDim.x * MT) {
    int col = p.colA[f];
    if (col < 0) {
      const unsigned int sf = tie_of((unsigned int)f);
      bool wins = true;
      unsigned int held = 0;
      for (int k = 0; k < 3; k++) {
        const int g = p.nbr[3 * (size_t)f + k];
        if (g < 0) continue;
        const int cg = p.colA[g];
        if (cg < 0) wins = wins && sf > tie_of((unsigned int)g);
        else held |= 1u << cg;
      }
      if (wins) {
        col = 0;
        while (held & (1u << col)) col++;
        top = max(top, col);
      } else {
        left++;
      }
    }
    p.colB[f] = col;
  }
  if (left) atomicAdd(&p.res->left, left);
  if (top >= 0) atomicMax(&p.res->maxColour, top);
}

// the labelled neighbours of f whose label differs from l
__device__ __forceinline__ int disagree(const TextureParams &p, int f, int l, bool above)
{
  int n = 0;
  for (int k = 0; k < 3; k++) {
    const int g = p.nbr[3 * (size_t)f + k];
    if (g < 0 || (above && g < f)) continue;
    const int lg = p.label[g];
    n += lg >= 0 && lg != l;
  }
  return n;
}

// e_f = D(f, l_f) + lambda * (the labelled neighbours g > f across an edge with l_g != l_f): tile partials
__global__ void __launch_bounds__(MT) texture_energy_kernel(TextureParams p)
{
  co_tree_tiles<1, MT>(p.T, p.part, [&](int f, double *v) {
    const int l = p.label[f];
    if (l < 0) return;
    const double *cq = p.cq + (size_t)f * MCAND;
    const int *ca = p.ca + (size_t)f * MCAND;
    int r = 0;
    while (ca[r] != l) r++;
    v[0] += (1.0 - cq[r] / cq[0]) + p.lambda * (double)disagree(p, f, l, true);
  });
}

// one CTA: the group partials and the total of the tile partials
__global__ void __launch_bounds__(MT) texture_total_kernel(TextureParams p)
{
  double tot[1];
  co_tree_groups<1, MT>(p.T, p.part, p.group);
  co_tree_total<1, MT>(p.T, p.group, tot);
  if (threadIdx.x == 0) p.res->energy = tot[0];
}

// An ICM step of the faces of one colour: the candidate of lowest local energy, the current label on ties, then the
// earlier rank.
__global__ void __launch_bounds__(MT) texture_icm_kernel(TextureParams p, int colour)
{
  unsigned int changed = 0;
  for (int f = blockIdx.x * MT + threadIdx.x; f < p.T; f += gridDim.x * MT) {
    const int cur = p.label[f];
    if (cur < 0 || p.colA[f] != colour) continue;
    const double *cq = p.cq + (size_t)f * MCAND;
    const int *ca = p.ca + (size_t)f * MCAND;
    const int m = p.cn[f] < MCAND ? p.cn[f] : MCAND;
    auto local = [&](int r) { return (1.0 - cq[r] / cq[0]) + p.lambda * (double)disagree(p, f, ca[r], false); };
    int r0 = 0;
    while (ca[r0] != cur) r0++;
    int best = cur;
    double bestE = local(r0);
    for (int r = 0; r < m; r++) {
      const double e = local(r);
      if (e < bestE) { bestE = e; best = ca[r]; }
    }
    if (best != cur) {
      p.label[f] = best;
      changed++;
    }
  }
  if (changed) atomicAdd(&p.res->changed, changed);
}

// ---- belief propagation of cs_texture_mesh_bp (rule 4b) -----------------------------------------------------------
// Min-sum messages over the Potts factors of the seen faces, a colour per step, then a decode.  Like the photo call's,
// the new words and fields travel as a second kernel argument.
struct BpResult {
  unsigned int changed;                       // messages with an entry that changed in a sweep
  unsigned int moved;                         // decoded labels that differ from the start label
};

struct BpParams {
  BpResult *res;
  double *msg;                                // [T][3][MCAND]: the message into f across its edge k, over f's ranks
};

// A step of the faces of one colour: every message out of every seen face of the colour, into the slot of the seen
// neighbour across the same edge.  It reads only the messages into faces of the colour, which no face of it writes.
__global__ void __launch_bounds__(MT) texture_bp_kernel(TextureParams p, BpParams b, int colour)
{
  unsigned int changed = 0;
  for (int f = blockIdx.x * MT + threadIdx.x; f < p.T; f += gridDim.x * MT) {
    const int m = p.cn[f];
    if (m <= 0 || p.colA[f] != colour) continue;
    const double *cq = p.cq + (size_t)f * MCAND;
    const int *ca = p.ca + (size_t)f * MCAND;
    const double *in = b.msg + (size_t)f * 3 * MCAND;
    for (int k = 0; k < 3; k++) {
      const int g = p.nbr[3 * (size_t)f + k];
      if (g < 0 || p.cn[g] <= 0) continue;
      // g's slot with f's edge k: the two vertex ids compared (rule 1 makes it unique)
      const int v0 = p.tin[3 * (size_t)f + k], v1 = p.tin[3 * (size_t)f + (k + 1) % 3];
      const int *tg = p.tin + 3 * (size_t)g;
      int kg = 0;
      while (!((tg[kg] == v0 && tg[(kg + 1) % 3] == v1) || (tg[kg] == v1 && tg[(kg + 1) % 3] == v0))) kg++;
      // h(r) = D(f, r) + the messages into f at the slots j != k, in ascending j
      double h[MCAND], hmin = 0.0;
      for (int r = 0; r < m; r++) {
        double s = 1.0 - cq[r] / cq[0];
        for (int j = 0; j < 3; j++)
          if (j != k) s = s + in[j * MCAND + r];
        h[r] = s;
        if (r == 0 || s < hmin) hmin = s;
      }
      const double jump = hmin + p.lambda;
      const int mg = p.cn[g];
      const int *cag = p.ca + (size_t)g * MCAND;
      double M[MCAND], Mmin = 0.0;
      for (int q = 0; q < mg; q++) {
        double x = jump;
        for (int r = 0; r < m; r++)
          if (ca[r] == cag[q] && h[r] < x) x = h[r];
        M[q] = x;
        if (q == 0 || x < Mmin) Mmin = x;
      }
      double *out = b.msg + ((size_t)g * 3 + kg) * MCAND;
      bool diff = false;
      for (int q = 0; q < mg; q++) {
        const double x = M[q] - Mmin;
        diff = diff || __double_as_longlong(out[q]) != __double_as_longlong(x);
        out[q] = x;
      }
      changed += diff;
    }
  }
  if (changed) atomicAdd(&b.res->changed, changed);
}

// The labels after a sweep: b_f(r) = D(f, r) + every message into f in ascending slot order, the lowest rank of
// minimum b; counts the labels that differ from the start label (rank 0).
__global__ void __launch_bounds__(MT) texture_bp_decode_kernel(TextureParams p, BpParams b)
{
  unsigned int moved = 0;
  for (int f = blockIdx.x * MT + threadIdx.x; f < p.T; f += gridDim.x * MT) {
    const int m = p.cn[f];
    if (m <= 0) continue;
    const double *cq = p.cq + (size_t)f * MCAND;
    const double *in = b.msg + (size_t)f * 3 * MCAND;
    int best = 0;
    double bestB = 0.0;
    for (int r = 0; r < m; r++) {
      const double s = (((1.0 - cq[r] / cq[0]) + in[r]) + in[MCAND + r]) + in[2 * MCAND + r];
      if (r == 0 || s < bestB) { bestB = s; best = r; }
    }
    p.label[f] = p.ca[(size_t)f * MCAND + best];
    moved += best != 0;
  }
  if (moved) atomicAdd(&b.res->moved, moved);
}

// ---- charts (rule 5) ----------------------------------------------------------------------------------------------
// union of every adjacent pair with equal labels (uf_link: every root is the lowest face of its component)
__global__ void __launch_bounds__(MT) texture_hook_kernel(TextureParams p)
{
  for (int f = blockIdx.x * MT + threadIdx.x; f < p.T; f += gridDim.x * MT) {
    const int l = p.label[f];
    if (l < 0) continue;
    for (int k = 0; k < 3; k++) {
      const int g = p.nbr[3 * (size_t)f + k];
      if (g <= f || p.label[g] != l) continue;
      uf_link(p.parent, f, g);
    }
  }
}

// colB[f] = the root of f.  Not into parent: a halving store of another thread's search could overwrite a root stored
// there with an ancestor that is not the root.  colB is free once the sweeps end; the host then passes it on as parent.
__global__ void __launch_bounds__(MT) texture_roots_kernel(TextureParams p)
{
  for (int f = blockIdx.x * MT + threadIdx.x; f <= p.T; f += gridDim.x * MT) {
    if (f == p.T) { p.flag[f] = 0; continue; }
    const int r = uf_find(p.parent, f);
    p.colB[f] = r;
    p.flag[f] = p.label[f] >= 0 && r == f;
  }
}

__global__ void __launch_bounds__(MT) texture_chart_init_kernel(TextureParams p)
{
  for (int f = blockIdx.x * MT + threadIdx.x; f < p.T; f += gridDim.x * MT) {
    if (!p.flag[f]) continue;
    int *e = p.craw + 6 * (size_t)p.chartIdx[f];
    e[0] = p.label[f];
    e[1] = e[2] = INT_MAX;
    e[3] = e[4] = INT_MIN;
    e[5] = 0;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) p.res->charts = p.chartIdx[p.T];
}

__global__ void __launch_bounds__(MT) texture_rect_kernel(TextureParams p)
{
  for (int f = blockIdx.x * MT + threadIdx.x; f < p.T; f += gridDim.x * MT) {
    const int l = p.label[f];
    if (l < 0) continue;
    int *e = p.craw + 6 * (size_t)p.chartIdx[p.parent[f]];
    const TexCam &c = p.cams[l];
    for (int k = 0; k < 3; k++) {
      double u, v, z;
      project(c, vertex_of(p.vin, p.tin[3 * (size_t)f + k]), u, v, z);
      atomicMin(e + 1, (int)floor(u));
      atomicMin(e + 2, (int)floor(v));
      atomicMax(e + 3, (int)ceil(u));
      atomicMax(e + 4, (int)ceil(v));
    }
    atomicAdd(e + 5, 1);
  }
}

// ---- outputs (rule 6) ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MT) texture_uv_kernel(TextureParams p)
{
  for (int f = blockIdx.x * MT + threadIdx.x; f < p.T; f += gridDim.x * MT) {
    const int l = p.label[f];
    float *uv = p.uv + 6 * (size_t)f;
    p.faceView[f] = l;
    if (l < 0) {
      for (int k = 0; k < 6; k++) uv[k] = __int_as_float(0x7fc00000);
      if (p.faceChart) p.faceChart[f] = -1;
      continue;
    }
    const int ch = p.chartIdx[p.parent[f]];
    const int *e = p.ctab + 8 * (size_t)ch;
    const TexCam &c = p.cams[l];
    for (int k = 0; k < 3; k++) {
      double u, v, z;
      project(c, vertex_of(p.vin, p.tin[3 * (size_t)f + k]), u, v, z);
      uv[2 * k] = __double2float_rn((u - (double)e[1]) + (double)e[5]);
      uv[2 * k + 1] = __double2float_rn((v - (double)e[2]) + (double)e[6]);
    }
    if (p.faceChart) p.faceChart[f] = ch;
  }
}

// one thread per chart texel (charts one after the other, rows of a chart in order)
__global__ void __launch_bounds__(MT) texture_atlas_kernel(TextureParams p)
{
  const long long n = p.numCharts ? p.cstart[p.numCharts] : 0;
  for (long long i = blockIdx.x * (long long)MT + threadIdx.x; i < n; i += (long long)gridDim.x * MT) {
    int lo = 0, hi = p.numCharts - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (p.cstart[mid] <= i) lo = mid; else hi = mid - 1;
    }
    const int *e = p.ctab + 8 * (size_t)lo;
    const int w = e[3];
    const long long local = i - p.cstart[lo];
    const int y = (int)(local / w), x = (int)(local - (long long)y * w);
    const int Y = e[6] + y;
    if (Y >= p.rowsWritten) continue;
    const TexCam &c = p.cams[e[0]];
    p.atlas[(size_t)Y * p.atlasWidth + e[5] + x] = c.img[(size_t)(e[2] + y) * c.pitch + e[1] + x];
  }
}

// where PhotoResult and BpResult start in the pinned readback buffer
size_t photo_result_at() { return (sizeof(TextureResult) + 15) & ~(size_t)15; }
size_t bp_result_at() { return (photo_result_at() + sizeof(PhotoResult) + 15) & ~(size_t)15; }

}  // namespace

int texture_run(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
                const float *vin, int V, const int *tin, int T, double lambda, double maxViewAngleDeg,
                double depthTol, int padding, int atlasWidth, int maxSweeps, float *atlas, int maxAtlasRows, float *uv,
                int *faceView, int *faceChart, int *chartsOut, int maxCharts, cudaStream_t st, void *h_res,
                double *info, long long *stats, const TexturePhoto *photo, int maxBpSweeps)
{
  const size_t C3 = 3 * (size_t)T;
  size_t tb[2] = {};
  CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb[0], (unsigned long long *)nullptr,
                                          (unsigned long long *)nullptr, (int *)nullptr, (int *)nullptr, (int)C3, 0,
                                          64, st));
  CS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb[1], (int *)nullptr, (int *)nullptr, T + 1, st));
  size_t tempBytes = std::max(tb[0], tb[1]);
  const long long cap = g_texture_group_bytes > 0 ? g_texture_group_bytes : TEXTURE_GROUP_BYTES;

  // the image groups: consecutive images while their buffers fit the cap (at least one image each)
  std::vector<int> groupStart{0};
  long long bufMax = 0, acc = 0;
  for (int a = 0; a < numImages; a++) {
    const long long b = 8ll * images[a].width * images[a].height;
    if (a > groupStart.back() && acc + b > cap) {
      groupStart.push_back(a);
      acc = 0;
    }
    acc += b;
    bufMax = std::max(bufMax, acc);
  }
  groupStart.push_back(numImages);
  const int tiles = (T + CO_TREE_TILE - 1) / CO_TREE_TILE, groups = (tiles + MT - 1) / MT;

  Layout L(256);
  const size_t resAt = L.take(sizeof(TextureResult));
  const size_t camAt = L.take((size_t)numImages * sizeof(TexCam));
  const size_t ekAt = L.take(C3 * 8), ekSAt = L.take(C3 * 8), evAt = L.take(C3 * 4), evSAt = L.take(C3 * 4);
  const size_t nbrAt = L.take(C3 * 4);
  const size_t cqAt = L.take((size_t)T * MCAND * 8), caAt = L.take((size_t)T * MCAND * 4), cnAt = L.take((size_t)T * 4);
  const size_t labAt = L.take((size_t)T * 4), colAAt = L.take((size_t)T * 4), colBAt = L.take((size_t)T * 4);
  const size_t parAt = L.take((size_t)T * 4), flagAt = L.take(((size_t)T + 1) * 4),
               idxAt = L.take(((size_t)T + 1) * 4);
  const size_t partAt = L.take((size_t)tiles * 8), groupAt = L.take((size_t)groups * 8);
  const size_t crawAt = L.take((size_t)T * 24), ctabAt = L.take((size_t)T * 32),
               cstartAt = L.take(((size_t)T + 1) * 8);
  const size_t bufAt = L.take((size_t)bufMax);
  const size_t tempAt = L.take(tempBytes);
  const size_t phResAt = photo ? L.take(sizeof(PhotoResult)) : 0, muAt = photo ? L.take((size_t)T * MCAND * 8) : 0;
  const bool withBp = maxBpSweeps >= 0;
  const size_t bpResAt = withBp ? L.take(sizeof(BpResult)) : 0, msgAt = withBp ? L.take((size_t)T * 3 * MCAND * 8) : 0,
               keptAt = withBp ? L.take((size_t)T * 4) : 0;
  char *base = nullptr;
  CS_CUDA(cudaMallocAsync((void **)&base, L.bytes, st));
  auto at = [&](size_t off) { return base + off; };

  std::vector<TexCam> cams(numImages);
  const double pi = 3.14159265358979323846;
  for (int a = 0; a < numImages; a++) {
    TexCam &c = cams[a];
    c.img = images[a].d_img;
    c.W = images[a].width;
    c.H = images[a].height;
    c.pitch = images[a].pitch;
    for (int k = 0; k < 9; k++) c.K[k] = Ks[9 * (size_t)a + k], c.R[k] = Rs[9 * (size_t)a + k];
    for (int k = 0; k < 3; k++) c.t[k] = ts[3 * (size_t)a + k];
    for (int i = 0; i < 3; i++) c.C[i] = -((c.R[i] * c.t[0] + c.R[3 + i] * c.t[1]) + c.R[6 + i] * c.t[2]);
    c.buf = nullptr;
  }

  TextureParams p{};
  p.res = reinterpret_cast<TextureResult *>(at(resAt));
  p.V = V;
  p.T = T;
  p.numImages = numImages;
  p.vin = vin;
  p.tin = tin;
  p.cams = reinterpret_cast<const TexCam *>(at(camAt));
  p.ekey = reinterpret_cast<unsigned long long *>(at(ekAt));
  p.ekeyS = reinterpret_cast<unsigned long long *>(at(ekSAt));
  p.eval = reinterpret_cast<int *>(at(evAt));
  p.evalS = reinterpret_cast<int *>(at(evSAt));
  p.nbr = reinterpret_cast<int *>(at(nbrAt));
  p.cq = reinterpret_cast<double *>(at(cqAt));
  p.ca = reinterpret_cast<int *>(at(caAt));
  p.cn = reinterpret_cast<int *>(at(cnAt));
  p.label = reinterpret_cast<int *>(at(labAt));
  p.colA = reinterpret_cast<int *>(at(colAAt));
  p.colB = reinterpret_cast<int *>(at(colBAt));
  p.parent = reinterpret_cast<int *>(at(parAt));
  p.flag = reinterpret_cast<int *>(at(flagAt));
  p.chartIdx = reinterpret_cast<int *>(at(idxAt));
  p.part = reinterpret_cast<double *>(at(partAt));
  p.group = reinterpret_cast<double *>(at(groupAt));
  p.lambda = lambda;
  p.cosLim = std::cos(maxViewAngleDeg * pi / 180.0);
  p.depthTol = depthTol;
  p.padding = padding;
  p.craw = reinterpret_cast<int *>(at(crawAt));
  p.ctab = reinterpret_cast<const int *>(at(ctabAt));
  p.cstart = reinterpret_cast<const long long *>(at(cstartAt));
  p.atlas = atlas;
  p.uv = uv;
  p.faceView = faceView;
  p.faceChart = faceChart;
  p.atlasWidth = atlasWidth;
  unsigned long long *buf = reinterpret_cast<unsigned long long *>(at(bufAt));
  void *temp = at(tempAt);
  TextureResult &R = *static_cast<TextureResult *>(h_res);
  PhotoParams ph{};
  PhotoResult *hPhoto = reinterpret_cast<PhotoResult *>(static_cast<char *>(h_res) + photo_result_at());
  if (photo) {
    ph.res = reinterpret_cast<PhotoResult *>(at(phResAt));
    ph.mu = reinterpret_cast<double *>(at(muAt));
    ph.dataTerm = photo->dataTerm;
    ph.outlierK = photo->outlierK;
    ph.minSigma = photo->outlierMinSigma;
    std::memset(hPhoto, 0, sizeof(PhotoResult));
  }
  BpParams bp{};
  BpResult *hBp = reinterpret_cast<BpResult *>(static_cast<char *>(h_res) + bp_result_at());
  int *kept = nullptr;
  if (withBp) {
    bp.res = reinterpret_cast<BpResult *>(at(bpResAt));
    bp.msg = reinterpret_cast<double *>(at(msgAt));
    kept = reinterpret_cast<int *>(at(keptAt));
  }
  cudaEvent_t *tev = match_timing_events();

  int status = 0, rounds = 0, sweeps = 0, colours = 0, bpSweeps = 0, bpKept = 0;
  long long changed = 0, fullRows = 0, rowsWritten = 0, bpChanged = 0, bpMoved = 0;
  double energy[3] = {0.0, 0.0, 0.0};
  std::vector<int> table;
  auto readback = [&]() -> int {
    CS_CUDA(cudaMemcpyAsync(h_res, p.res, sizeof(TextureResult), cudaMemcpyDeviceToHost, st));
    if (withBp) CS_CUDA(cudaMemcpyAsync(hBp, bp.res, sizeof(BpResult), cudaMemcpyDeviceToHost, st));
    CS_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  auto total = [&](double &out) -> int {
    texture_energy_kernel<<<grid_of(T), MT, 0, st>>>(p);
    texture_total_kernel<<<1, MT, 0, st>>>(p);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    int r;
    if ((r = readback()) < 0) return r;
    out = R.energy;
    return 0;
  };
  auto run = [&]() -> int {
    int r;
    if (tev) CS_CUDA(cudaEventRecord(tev[0], st));
    CS_CUDA(cudaMemsetAsync(p.res, 0, sizeof(TextureResult), st));
    if (withBp) CS_CUDA(cudaMemsetAsync(bp.res, 0, sizeof(BpResult), st));
    mesh_validate_kernel<<<grid_of(T), MT, 0, st>>>(vin, V, tin, T, &p.res->bad);
    count_launch();
    CS_CUDA(cudaGetLastError());
    if ((r = readback()) < 0) return r;
    if (R.bad) {
      status = 2;
      return 0;
    }
    texture_edges_kernel<<<grid_of(3ll * T), MT, 0, st>>>(p);
    CS_CUDA(cub::DeviceRadixSort::SortPairs(temp, tempBytes, p.ekey, p.ekeyS, p.eval, p.evalS, (int)C3, 0, 64, st));
    texture_adjacency_kernel<<<grid_of(3ll * T), MT, 0, st>>>(p);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    CS_CUDA(cudaMemsetAsync(p.cn, 0, (size_t)T * 4, st));
    if (photo) CS_CUDA(cudaMemsetAsync(ph.res, 0, sizeof(PhotoResult), st));
    if (tev) CS_CUDA(cudaEventRecord(tev[1], st));
    for (size_t gi = 0; gi + 1 < groupStart.size(); gi++) {
      const int g0 = groupStart[gi], g1 = groupStart[gi + 1];
      size_t off = 0;
      for (int a = g0; a < g1; a++) {
        cams[a].buf = buf + off;
        off += (size_t)images[a].width * images[a].height;
      }
      CS_CUDA(cudaMemcpyAsync(at(camAt), cams.data(), (size_t)numImages * sizeof(TexCam), cudaMemcpyHostToDevice, st));
      CS_CUDA(cudaMemsetAsync(buf, 0xff, off * 8, st));
      p.g0 = g0;
      p.gn = g1 - g0;
      texture_raster_kernel<<<grid_of((long long)p.gn * T), MT, 0, st>>>(p);
      if (tev && gi == 0) CS_CUDA(cudaEventRecord(tev[2], st));
      if (photo) texture_photo_candidate_kernel<<<grid_of(32ll * T), MT, 0, st>>>(p, ph);
      else texture_candidate_kernel<<<grid_of(T), MT, 0, st>>>(p);
      count_launch(2);
      CS_CUDA(cudaGetLastError());
      // the host table is read by the copy above before the next group changes it
      CS_CUDA(cudaStreamSynchronize(st));
    }
    if (photo) {
      texture_outlier_kernel<<<grid_of(T), MT, 0, st>>>(p, ph);
      count_launch();
      CS_CUDA(cudaGetLastError());
    }
    if (tev) CS_CUDA(cudaEventRecord(tev[3], st));
    texture_label_init_kernel<<<grid_of(T), MT, 0, st>>>(p);
    count_launch();
    CS_CUDA(cudaGetLastError());
    for (;;) {
      CS_CUDA(cudaMemsetAsync(&p.res->left, 0, sizeof(unsigned int), st));
      texture_colour_kernel<<<grid_of(T), MT, 0, st>>>(p);
      count_launch();
      CS_CUDA(cudaGetLastError());
      std::swap(p.colA, p.colB);
      rounds++;
      if ((r = readback()) < 0) return r;
      if (R.left == 0) break;
    }
    colours = R.maxColour + 1;
    if ((r = total(energy[0])) < 0) return r;
    // rule 4b: BP sweeps from zero messages, the labelling of lowest E kept (the start labelling first)
    energy[2] = energy[0];
    if (maxBpSweeps > 0) {
      CS_CUDA(cudaMemsetAsync(bp.msg, 0, (size_t)T * 3 * MCAND * 8, st));
      CS_CUDA(cudaMemcpyAsync(kept, p.label, (size_t)T * 4, cudaMemcpyDeviceToDevice, st));
      while (bpSweeps < maxBpSweeps) {
        CS_CUDA(cudaMemsetAsync(bp.res, 0, sizeof(BpResult), st));
        for (int c = 0; c < colours; c++) texture_bp_kernel<<<grid_of(T), MT, 0, st>>>(p, bp, c);
        texture_bp_decode_kernel<<<grid_of(T), MT, 0, st>>>(p, bp);
        count_launch(colours + 1);
        CS_CUDA(cudaGetLastError());
        double e;
        if ((r = total(e)) < 0) return r;
        bpSweeps++;
        bpChanged = hBp->changed;
        if (e < energy[2]) {
          energy[2] = e;
          bpKept = bpSweeps;
          bpMoved = hBp->moved;
          CS_CUDA(cudaMemcpyAsync(kept, p.label, (size_t)T * 4, cudaMemcpyDeviceToDevice, st));
        }
        if (bpChanged == 0) break;
      }
      if (bpKept != bpSweeps) CS_CUDA(cudaMemcpyAsync(p.label, kept, (size_t)T * 4, cudaMemcpyDeviceToDevice, st));
    }
    for (;;) {
      if (sweeps == maxSweeps) { status = 3; break; }
      CS_CUDA(cudaMemsetAsync(&p.res->changed, 0, sizeof(unsigned int), st));
      for (int c = 0; c < colours; c++) texture_icm_kernel<<<grid_of(T), MT, 0, st>>>(p, c);
      count_launch(colours);
      CS_CUDA(cudaGetLastError());
      sweeps++;
      if ((r = readback()) < 0) return r;
      changed += R.changed;
      if (R.changed == 0) { status = 0; break; }
    }
    if ((r = total(energy[1])) < 0) return r;
    if (tev) CS_CUDA(cudaEventRecord(tev[4], st));
    texture_hook_kernel<<<grid_of(T), MT, 0, st>>>(p);
    texture_roots_kernel<<<grid_of(T + 1ll), MT, 0, st>>>(p);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    std::swap(p.parent, p.colB);              // from here on every face's parent is its root
    CS_CUDA(cub::DeviceScan::ExclusiveSum(temp, tempBytes, p.flag, p.chartIdx, T + 1, st));
    texture_chart_init_kernel<<<grid_of(T), MT, 0, st>>>(p);
    texture_rect_kernel<<<grid_of(T), MT, 0, st>>>(p);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    if ((r = readback()) < 0) return r;
    const int C = R.charts;
    std::vector<int> raw(6 * (size_t)C);
    if (C) {
      CS_CUDA(cudaMemcpyAsync(raw.data(), p.craw, raw.size() * 4, cudaMemcpyDeviceToHost, st));
      CS_CUDA(cudaStreamSynchronize(st));
    }
    // the chart table, then the shelves (rule 6)
    table.assign(8 * (size_t)C, 0);
    for (int c = 0; c < C; c++) {
      const int *e = &raw[6 * (size_t)c];
      int *o = &table[8 * (size_t)c];
      const cs_image &I = images[e[0]];
      const int x0 = std::max(0, e[1] - padding), x1 = std::min(I.width - 1, e[3] + padding);
      const int y0 = std::max(0, e[2] - padding), y1 = std::min(I.height - 1, e[4] + padding);
      o[0] = e[0];
      o[1] = x0;
      o[2] = y0;
      o[3] = x1 - x0 + 1;
      o[4] = y1 - y0 + 1;
      o[7] = e[5];
    }
    std::vector<int> order(C);
    for (int c = 0; c < C; c++) order[c] = c;
    std::sort(order.begin(), order.end(), [&](int a, int b) {
      const int *x = &table[8 * (size_t)a], *y = &table[8 * (size_t)b];
      if (x[4] != y[4]) return x[4] > y[4];
      if (x[3] != y[3]) return x[3] > y[3];
      return a < b;
    });
    long long shelfY = 0, shelfH = 0, cx = 0;
    for (int c : order) {
      int *o = &table[8 * (size_t)c];
      if (cx + o[3] > atlasWidth) {
        shelfY += shelfH;
        shelfH = 0;
        cx = 0;
      }
      o[5] = (int)cx;
      o[6] = (int)shelfY;
      cx += o[3];
      shelfH = std::max(shelfH, (long long)o[4]);
    }
    fullRows = shelfY + shelfH;
    rowsWritten = std::min(fullRows, (long long)maxAtlasRows);
    std::vector<long long> starts((size_t)C + 1, 0);
    for (int c = 0; c < C; c++) starts[c + 1] = starts[c] + (long long)table[8 * (size_t)c + 3] * table[8 * (size_t)c + 4];
    if (C) {
      CS_CUDA(cudaMemcpyAsync(at(ctabAt), table.data(), table.size() * 4, cudaMemcpyHostToDevice, st));
      CS_CUDA(cudaMemcpyAsync(at(cstartAt), starts.data(), starts.size() * 8, cudaMemcpyHostToDevice, st));
    }
    p.numCharts = C;
    p.rowsWritten = (int)rowsWritten;
    if (tev) CS_CUDA(cudaEventRecord(tev[5], st));
    if (rowsWritten) CS_CUDA(cudaMemsetAsync(atlas, 0, (size_t)rowsWritten * atlasWidth * 4, st));
    texture_uv_kernel<<<grid_of(T), MT, 0, st>>>(p);
    texture_atlas_kernel<<<grid_of(starts[C]), MT, 0, st>>>(p);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    if (tev) CS_CUDA(cudaEventRecord(tev[6], st));
    if (photo) CS_CUDA(cudaMemcpyAsync(hPhoto, ph.res, sizeof(PhotoResult), cudaMemcpyDeviceToHost, st));
    CS_CUDA(cudaStreamSynchronize(st));
    if (tev) {
      static const char *const names[6] = {"adjacency", "depth", "candidates", "labelling", "charts", "atlas"};
      report_stage_times(tev, names, 6, "texture timing faces=%d images=%d groups=%d", T, numImages,
                         (int)groupStart.size() - 1);
    }
    return 0;
  };
  const int r = run();
  cudaFreeAsync(base, st);
  if (r < 0) return r;
  const bool out = status != 2;
  const int C = out ? R.charts : 0;
  for (int c = 0; c < std::min(C, maxCharts); c++)
    std::memcpy(chartsOut + 8 * (size_t)c, &table[8 * (size_t)c], 8 * sizeof(int));
  if (info) {
    info[0] = out ? energy[0] : 0.0;
    info[1] = out ? energy[1] : 0.0;
    if (withBp) info[2] = out ? energy[2] : 0.0;
  }
  if (stats) {
    stats[0] = T;
    stats[1] = out ? R.unseen : 0;
    stats[2] = out ? R.cand : 0;
    stats[3] = out ? colours : 0;
    stats[4] = rounds;
    stats[5] = sweeps;
    stats[6] = changed;
    stats[7] = C;
    stats[8] = fullRows;
    stats[9] = rowsWritten;
    stats[10] = status;
    if (photo) {
      stats[11] = out ? (long long)hPhoto->samples : 0;
      stats[12] = out ? (long long)hPhoto->fallbacks : 0;
      stats[13] = out ? hPhoto->tested : 0;
      stats[14] = out ? hPhoto->removed : 0;
      stats[15] = out ? hPhoto->bestRemoved : 0;
    }
    if (withBp) {
      stats[16] = bpSweeps;
      stats[17] = bpKept;
      stats[18] = bpChanged;
      stats[19] = bpMoved;
    }
  }
  return C;
}

// the photo call's counters follow TextureResult in the pinned readback buffer, and the BP call's follow those
size_t texture_result_bytes() { return bp_result_at() + sizeof(BpResult); }

}  // namespace cs
