// rotavg.cu -- rotation averaging over a view graph (cs_rotation_averaging).  The rules (spanning-tree start, residual,
// IRLS weights, the Laplacian system and its CG solve, the update, the stop rule, the outputs and the summation orders)
// are stated in cudasift_b200.h at cs_rotation_averaging; tests/rotavg_oracle.py restates them in float64.
//
// The spanning tree and the start rotations are host work (rotavg_prepare).  One counted launch follows:
//   (cub stable radix sort of the incidences (image, 2 e + side): every image's edges in edge order)
//   rotavg_kernel: one cooperative launch runs the whole IRLS loop, phases separated by grid barriers
// Every floating-point sum has a fixed order that depends on the data only (coop.cuh): per image, the pieces of the
// sorted incidences' tiles; totals over tiles of 256 edges (the cost) or 32 images (the CG dot products).  The largest
// step is a max, exact in any order.
// No floating-point atomics.  Every branch around a grid barrier (the CG stop, the IRLS stop) is taken on values that
// every CTA computes from the same words, written before the barrier, by the same instructions in the same order, so
// every CTA takes the same path; every loop is bounded by maxIterations or maxLinearIterations.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <numeric>
#include <vector>
#include <cooperative_groups.h>
#include <cub/cub.cuh>
#include <math_constants.h>

#include "common.cuh"
#include "coop.cuh"

namespace cg = cooperative_groups;

namespace cs {

namespace {

constexpr int RA_THREADS = 256;
constexpr int RA_PV = 4;             // an image piece: the sum of w, then three more (b, or the neighbours' w p)
// Slots per image tile partial: r.r (or b.b), r.z and p.q; p.q has a slot of its own, as in bundle.cu.
constexpr int RA_NP = 3;
constexpr double RA_STOP = 1e-12;    // radians: the IRLS loop stops once no image moves further

// An image: its rotation, its CG vectors (the world-frame tangent x and the CG state), the Laplacian diagonal and its
// sorted incidences [start, end).  free: reached and not the reference; reached: joined to the reference by the tree.
struct RaNode {
  double R[9];
  double x[3], r[3], z[3], p[3], q[3];
  double diag;
  int start, end, free, reached;
};

// An edge {i, j}: its relative rotation and weight; its residual and IRLS weight at the current rotations.  active:
// both images reached.
struct RaEdge {
  double Q[9];
  double rho[3];
  double w0, w;
  int i, j, active, pad;
};

static_assert(sizeof(RaNode) == 216 && sizeof(RaEdge) == 128, "the header states the scratch");

// The words the host reads back.
struct RaResult {
  double cost[2];
  unsigned long long iters, cgIters;
};

struct RaParams {
  RaNode *nodes;
  RaEdge *edges;
  double *theta;                     // [numEdges]: the final residual angle (radians; NaN for an inactive edge)
  const int *keysS, *order;          // [2 numEdges]: the incidences sorted by image
  double *pieces;                    // [tiles + numImages][RA_PV]
  double *nodePart;                  // [ceil(numImages / 32)][RA_NP]
  double *maxPart;                   // [ceil(numImages / 32)]
  double *edgePart;                  // [ceil(numEdges / 256)]
  double *trace;                     // [maxIterations][3]
  RaResult *res;
  double sigma2, tol2;
  int numImages, numEdges, maxIterations, maxLinear;
};

// The rotation vector of D (log), returned angle theta = atan2(s, c) with c = (tr D - 1) / 2 and s = |v|, v the axial
// vector of (D - D^T) / 2.  For c > 0 the vector is v theta / s (v when s = 0); otherwise it is theta a, a the unit
// axis from the symmetric part (D + D^T) / 2 = c I + (1 - c) a a^T through its largest diagonal entry, signed so that
// a.v >= 0.
__host__ __device__ inline double ra_log(const double (&D)[9], double (&w)[3])
{
  const double c = 0.5 * (D[0] + D[4] + D[8] - 1.0);
  const double v[3] = {0.5 * (D[7] - D[5]), 0.5 * (D[2] - D[6]), 0.5 * (D[3] - D[1])};
  const double s = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  const double th = atan2(s, c);
  if (c > 0.0) {
    const double f = s > 0.0 ? th / s : 1.0;
    for (int i = 0; i < 3; i++) w[i] = f * v[i];
    return th;
  }
  const int k = D[4] > D[0] ? (D[8] > D[4] ? 2 : 1) : (D[8] > D[0] ? 2 : 0);
  const double u = 1.0 - c;
  double a[3];
  a[k] = sqrt(fmax(D[4 * k] - c, 0.0) / u);
  for (int m = 0; m < 3; m++)
    if (m != k) a[m] = 0.5 * (D[3 * k + m] + D[3 * m + k]) / (u * a[k]);
  const double sg = a[0] * v[0] + a[1] * v[1] + a[2] * v[2] < 0.0 ? -th : th;
  for (int i = 0; i < 3; i++) w[i] = sg * a[i];
  return th;
}

// Edge e at the current rotations: rho = log(R_j^T Q R_i), the IRLS weight and the cost term (header: the loss).
__device__ __forceinline__ double ra_edge(const RaParams &p, int e)
{
  RaEdge &g = p.edges[e];
  if (!g.active) {
    p.theta[e] = CUDART_NAN;
    return 0.0;
  }
  const double *Ri = p.nodes[g.i].R, *Rj = p.nodes[g.j].R;
  double QR[9], D[9], rho[3];
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++) QR[3 * a + b] = g.Q[3 * a] * Ri[b] + g.Q[3 * a + 1] * Ri[3 + b] + g.Q[3 * a + 2] * Ri[6 + b];
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++) D[3 * a + b] = Rj[a] * QR[b] + Rj[3 + a] * QR[3 + b] + Rj[6 + a] * QR[6 + b];
  const double th = ra_log(D, rho), t2 = th * th;
  const double q = p.sigma2 > 0.0 ? p.sigma2 / (t2 + p.sigma2) : 1.0;
#pragma unroll
  for (int k = 0; k < 3; k++) g.rho[k] = rho[k];
  g.w = g.w0 * (q * q);
  p.theta[e] = th;
  return g.w0 * (t2 * q);
}

// The largest of n non-negative tile maxima, in every thread of the CTA (a max of non-negative doubles is the max of
// their bit patterns).
__device__ __forceinline__ double ra_max_total(const double *part, int n)
{
  __shared__ unsigned long long s_max;
  if (threadIdx.x < 32) {
    unsigned long long m = 0;
    for (int i = (int)threadIdx.x; i < n; i += 32) m = max(m, (unsigned long long)__double_as_longlong(part[i]));
    m = vp_warp_max(m);
    if (threadIdx.x == 0) s_max = m;
  }
  __syncthreads();
  const double out = __longlong_as_double((long long)s_max);
  __syncthreads();
  return out;
}

__global__ void __launch_bounds__(RA_THREADS) rotavg_kernel(RaParams p)
{
  cg::grid_group grid = cg::this_grid();
  const int tid = (int)(blockIdx.x * RA_THREADS + threadIdx.x), nthreads = (int)gridDim.x * RA_THREADS;
  const int lane = (int)threadIdx.x & 31, warpG = tid >> 5, numWarps = nthreads >> 5;
  const int C = p.numImages, n = 2 * p.numEdges;
  const int nodeTiles = (C + 31) / 32, edgeTiles = (p.numEdges + RA_THREADS - 1) / RA_THREADS;

  // 0. every image's sorted incidences; the residuals at the start rotations and their cost
  co_ranges(p.keysS, n, p.nodes, tid, nthreads);
  co_per_item<1, RA_THREADS>(p.numEdges, p.edgePart, [&](int e, double *v) { v[0] = ra_edge(p, e); });
  grid.sync();
  double cost;
  {
    double t[1];
    co_totals<1>(p.edgePart, edgeTiles, 1, t);
    cost = t[0];
  }
  const double cost0 = cost;
  unsigned long long iters = 0, cgTotal = 0;

  for (int it = 0; it < p.maxIterations; it++) {
    iters++;
    // A. the image pieces: the Laplacian diagonal sum w and b = sum over its edges of -w rho (as i) or +w rho (as j)
    co_pieces<4, 0, RA_PV, RA_THREADS>(p.keysS, p.order, p.pieces, n, p.nodes, [&](int code, int, double *v) {
      const RaEdge &g = p.edges[code >> 1];
      const double sg = (code & 1) ? g.w : -g.w;
      v[0] = g.w;
#pragma unroll
      for (int k = 0; k < 3; k++) v[1 + k] = sg * g.rho[k];
    });
    grid.sync();

    // B. per image (a lane each): x = 0, r = b, z = r / diag, p = 0 (held images: all zero); the partials of b.b, r.z
    for (int w = warpG; w < nodeTiles; w += numWarps) {
      const int a = w * 32 + lane;
      double d[2] = {0.0, 0.0};
      if (a < C) {
        RaNode &c = p.nodes[a];
        double G[4];
        co_gather<4, 0, RA_PV>(p.pieces, a, c, G);
        c.diag = G[0];
        const double inv = c.free && G[0] > 0.0 ? 1.0 / G[0] : 0.0;
#pragma unroll
        for (int k = 0; k < 3; k++) {
          const double r = c.free ? G[1 + k] : 0.0, z = r * inv;
          c.x[k] = 0.0; c.r[k] = r; c.z[k] = z; c.p[k] = 0.0;
          d[0] += r * r;
          d[1] += r * z;
        }
      }
      co_warp_partial<2>(d, p.nodePart + RA_NP * (size_t)w);
    }
    grid.sync();

    // C-F. Jacobi-preconditioned CG on L x = b from x = 0
    int cgIt = 0;
    {
      double t2[2];
      co_totals<2>(p.nodePart, nodeTiles, RA_NP, t2);
      const double thr = p.tol2 * t2[0];
      double rr = t2[0], rz = t2[1], beta = 0.0;
      while (cgIt < p.maxLinear && !(rr <= thr)) {
        // C. the image pieces of sum over its edges of w p_other, p = z + beta p_old of the other image
        co_pieces<3, 1, RA_PV, RA_THREADS>(p.keysS, p.order, p.pieces, n, p.nodes, [&](int code, int, double *v) {
          const RaEdge &g = p.edges[code >> 1];
          const RaNode &o = p.nodes[(code & 1) ? g.i : g.j];
#pragma unroll
          for (int k = 0; k < 3; k++) v[k] = g.w * fma(beta, o.p[k], o.z[k]);
        });
        grid.sync();
        // D. per image: p = z + beta p_old, q = L p = diag p - sum w p_other (held images 0); the partials of p.q
        for (int w = warpG; w < nodeTiles; w += numWarps) {
          const int a = w * 32 + lane;
          double d[1] = {0.0};
          if (a < C) {
            RaNode &c = p.nodes[a];
            double Wp[3];
            co_gather<3, 1, RA_PV>(p.pieces, a, c, Wp);
#pragma unroll
            for (int k = 0; k < 3; k++) {
              const double pn = fma(beta, c.p[k], c.z[k]);
              const double q = c.free ? c.diag * pn - Wp[k] : 0.0;
              c.p[k] = pn;
              c.q[k] = q;
              d[0] += pn * q;
            }
          }
          co_warp_partial<1>(d, p.nodePart + RA_NP * (size_t)w + 2);
        }
        grid.sync();
        double pq[1];
        co_totals<1>(p.nodePart + 2, nodeTiles, RA_NP, pq);
        if (!(pq[0] > 0.0)) break;
        const double alpha = rz / pq[0];
        // E. per image: x += alpha p, r -= alpha q, z = r / diag; the partials of r.r and r.z
        for (int w = warpG; w < nodeTiles; w += numWarps) {
          const int a = w * 32 + lane;
          double d[2] = {0.0, 0.0};
          if (a < C) {
            RaNode &c = p.nodes[a];
            const double inv = c.free && c.diag > 0.0 ? 1.0 / c.diag : 0.0;
#pragma unroll
            for (int k = 0; k < 3; k++) {
              c.x[k] = fma(alpha, c.p[k], c.x[k]);
              const double r = fma(-alpha, c.q[k], c.r[k]), z = r * inv;
              c.r[k] = r;
              c.z[k] = z;
              d[0] += r * r;
              d[1] += r * z;
            }
          }
          co_warp_partial<2>(d, p.nodePart + RA_NP * (size_t)w);
        }
        cgIt++;
        grid.sync();
        co_totals<2>(p.nodePart, nodeTiles, RA_NP, t2);
        rr = t2[0];
        beta = t2[1] / rz;
        rz = t2[1];
      }
    }
    cgTotal += cgIt;

    // G. per free image: R <- exp([R x]x) R (= R exp([x]x), x in the world frame); the tile maxima of |x|
    for (int w = warpG; w < nodeTiles; w += numWarps) {
      const int a = w * 32 + lane;
      unsigned long long m = 0;
      if (a < C && p.nodes[a].free) {
        RaNode &c = p.nodes[a];
        const double len = sqrt(c.x[0] * c.x[0] + c.x[1] * c.x[1] + c.x[2] * c.x[2]);
        double wc[3], R1[9], Q[9];
#pragma unroll
        for (int k = 0; k < 3; k++) wc[k] = c.R[3 * k] * c.x[0] + c.R[3 * k + 1] * c.x[1] + c.R[3 * k + 2] * c.x[2];
        vp_rotate(wc, c.R, R1, Q);
#pragma unroll
        for (int k = 0; k < 9; k++) c.R[k] = R1[k];
        m = (unsigned long long)__double_as_longlong(len);
      }
      m = vp_warp_max(m);
      if (lane == 0) p.maxPart[w] = __longlong_as_double((long long)m);
    }
    grid.sync();
    const double step = ra_max_total(p.maxPart, nodeTiles);

    // H. the residuals at the new rotations; the trace row
    co_per_item<1, RA_THREADS>(p.numEdges, p.edgePart, [&](int e, double *v) { v[0] = ra_edge(p, e); });
    grid.sync();
    if (tid == 0) {
      double *tr = p.trace + 3 * (size_t)it;
      tr[0] = cost;
      tr[1] = (double)cgIt;
      tr[2] = step;
    }
    {
      double t[1];
      co_totals<1>(p.edgePart, edgeTiles, 1, t);
      cost = t[0];
    }
    if (step <= RA_STOP) break;
  }
  if (tid == 0) {
    p.res->cost[0] = cost0;
    p.res->cost[1] = cost;
    p.res->iters = iters;
    p.res->cgIters = cgTotal;
  }
}

// The pinned layout: the result words, the trace, the image and edge tables, the incidence keys and values, the final
// angles.
struct RaHost {
  size_t traceAt, nodeAt, edgeAt, keysAt, valsAt, thetaAt, bytes;
  RaHost(int numImages, int numEdges, int maxIterations)
  {
    Layout H(256);
    H.take(sizeof(RaResult));
    traceAt = H.take((size_t)maxIterations * 3 * sizeof(double));
    nodeAt = H.take((size_t)numImages * sizeof(RaNode));
    edgeAt = H.take((size_t)numEdges * sizeof(RaEdge));
    keysAt = H.take((size_t)numEdges * 2 * sizeof(int));
    valsAt = H.take((size_t)numEdges * 2 * sizeof(int));
    thetaAt = H.take((size_t)numEdges * sizeof(double));
    bytes = H.bytes;
  }
};

void mat_mul(const double *A, const double *B, double *C, bool transA)
{
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) {
      double s = 0.0;
      for (int k = 0; k < 3; k++) s += (transA ? A[3 * k + a] : A[3 * a + k]) * B[3 * k + b];
      C[3 * a + b] = s;
    }
}

}  // namespace

int rotavg_prepare(DeviceCtx &c, int numImages, const int *edges, int numEdges, const double *Rrel,
                   const double *weights, int refImage, int maxIterations)
{
  const RaHost H(numImages, numEdges, maxIterations);
  int r = c.h_rotavg.grow(H.bytes);
  if (r < 0) return r;
  char *base = c.h_rotavg.as<char>();
  RaNode *nodes = reinterpret_cast<RaNode *>(base + H.nodeAt);
  RaEdge *eds = reinterpret_cast<RaEdge *>(base + H.edgeAt);
  int *keys = reinterpret_cast<int *>(base + H.keysAt), *vals = reinterpret_cast<int *>(base + H.valsAt);
  memset(nodes, 0, (size_t)numImages * sizeof(RaNode));

  // Kruskal: edges by weight descending, ties to the lower index; union-find with path halving and union by size
  std::vector<int> byWeight(numEdges), parent(numImages), size(numImages, 1);
  std::iota(byWeight.begin(), byWeight.end(), 0);
  std::stable_sort(byWeight.begin(), byWeight.end(), [&](int a, int b) { return weights[a] > weights[b]; });
  std::iota(parent.begin(), parent.end(), 0);
  auto root = [&](int x) {
    while (parent[x] != x) x = parent[x] = parent[parent[x]];
    return x;
  };
  std::vector<char> inTree(numEdges, 0);
  std::vector<int> degree(numImages + 1, 0);
  for (int e : byWeight) {
    int a = root(edges[2 * e]), b = root(edges[2 * e + 1]);
    if (a == b) continue;
    if (size[a] < size[b]) std::swap(a, b);
    parent[b] = a;
    size[a] += size[b];
    inTree[e] = 1;
    degree[edges[2 * e]]++;
    degree[edges[2 * e + 1]]++;
  }
  // the tree's adjacency in ascending edge order, then a BFS from the reference
  std::vector<int> adjAt(numImages + 1, 0), adj;
  for (int a = 0; a < numImages; a++) adjAt[a + 1] = adjAt[a] + degree[a];
  adj.resize(adjAt[numImages]);
  std::vector<int> fill(adjAt.begin(), adjAt.end() - 1);
  for (int e = 0; e < numEdges; e++)
    if (inTree[e]) {
      adj[fill[edges[2 * e]]++] = e;
      adj[fill[edges[2 * e + 1]]++] = e;
    }
  std::vector<int> queue;
  queue.reserve(numImages);
  queue.push_back(refImage);
  RaNode &ref = nodes[refImage];
  for (int k = 0; k < 9; k++) ref.R[k] = (k % 4 == 0) ? 1.0 : 0.0;
  ref.reached = 1;
  for (size_t h = 0; h < queue.size(); h++) {
    const int a = queue[h];
    for (int k = adjAt[a]; k < adjAt[a + 1]; k++) {
      const int e = adj[k], i = edges[2 * e], j = edges[2 * e + 1], o = i == a ? j : i;
      if (nodes[o].reached) continue;
      // R_j = Q R_i from i, R_i = Q^T R_j from j
      mat_mul(Rrel + 9 * (size_t)e, nodes[a].R, nodes[o].R, o == i);
      nodes[o].reached = 1;
      nodes[o].free = 1;
      queue.push_back(o);
    }
  }
  for (int e = 0; e < numEdges; e++) {
    RaEdge &g = eds[e];
    memset(&g, 0, sizeof g);
    for (int k = 0; k < 9; k++) g.Q[k] = Rrel[9 * (size_t)e + k];
    g.w0 = weights[e];
    g.i = edges[2 * e];
    g.j = edges[2 * e + 1];
    g.active = nodes[g.i].reached;
    keys[2 * e] = g.i;
    keys[2 * e + 1] = g.j;
    vals[2 * e] = 2 * e;
    vals[2 * e + 1] = 2 * e + 1;
  }
  return 0;
}

int rotavg_enqueue(DeviceCtx &c, int numImages, int numEdges, int maxIterations, int maxLinearIterations,
                   double linearTol, double sigmaDeg)
{
  const int C = numImages, E = numEdges, n = 2 * E;
  const int tiles = idivup(n, CO_TILE);
  const int bits = radix_bits(C - 1);                              // every key is < C
  size_t sortBytes = 0;
  CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sortBytes, (int *)nullptr, (int *)nullptr, (int *)nullptr,
                                          (int *)nullptr, n, 0, bits, c.stream));
  // device scratch (header: cs_rotation_averaging)
  Layout L(256);
  const size_t resAt = L.take(sizeof(RaResult)), traceAt = L.take((size_t)maxIterations * 3 * sizeof(double));
  const size_t zeroEnd = L.bytes;
  const size_t nodeAt = L.take((size_t)C * sizeof(RaNode)), edgeAt = L.take((size_t)E * sizeof(RaEdge));
  const size_t thetaAt = L.take((size_t)E * sizeof(double));
  const size_t keysAt = L.take((size_t)n * sizeof(int)), valsAt = L.take((size_t)n * sizeof(int));
  const size_t keysSAt = L.take((size_t)n * sizeof(int)), orderAt = L.take((size_t)n * sizeof(int));
  const size_t piecesAt = L.take(((size_t)tiles + C) * RA_PV * sizeof(double));
  const size_t nodePartAt = L.take((size_t)idivup(C, 32) * RA_NP * sizeof(double));
  const size_t maxPartAt = L.take((size_t)idivup(C, 32) * sizeof(double));
  const size_t edgePartAt = L.take((size_t)idivup(E, RA_THREADS) * sizeof(double));
  const size_t tempAt = L.take(sortBytes);
  int r = c.rotavg.grow(L.bytes);
  if (r < 0) return r;
  char *base = c.rotavg.as<char>();
  const RaHost H(C, E, maxIterations);
  const char *hb = c.h_rotavg.as<const char>();

  RaParams prm;
  prm.res = reinterpret_cast<RaResult *>(base + resAt);
  prm.trace = reinterpret_cast<double *>(base + traceAt);
  prm.nodes = reinterpret_cast<RaNode *>(base + nodeAt);
  prm.edges = reinterpret_cast<RaEdge *>(base + edgeAt);
  prm.theta = reinterpret_cast<double *>(base + thetaAt);
  prm.keysS = reinterpret_cast<const int *>(base + keysSAt);
  prm.order = reinterpret_cast<const int *>(base + orderAt);
  prm.pieces = reinterpret_cast<double *>(base + piecesAt);
  prm.nodePart = reinterpret_cast<double *>(base + nodePartAt);
  prm.maxPart = reinterpret_cast<double *>(base + maxPartAt);
  prm.edgePart = reinterpret_cast<double *>(base + edgePartAt);
  const double sigma = sigmaDeg * (CUDART_PI / 180.0);
  prm.sigma2 = sigma * sigma;
  prm.tol2 = linearTol * linearTol;
  prm.numImages = C;
  prm.numEdges = E;
  prm.maxIterations = maxIterations;
  prm.maxLinear = maxLinearIterations;

  const int wave = coop_grid<rotavg_kernel, RA_THREADS>("cs_rotation_averaging");
  if (wave < 0) return wave;
  const cudaStream_t st = c.stream;
  CS_CUDA(cudaMemsetAsync(base, 0, zeroEnd, st));
  CS_CUDA(cudaMemcpyAsync(prm.nodes, hb + H.nodeAt, (size_t)C * sizeof(RaNode), cudaMemcpyHostToDevice, st));
  CS_CUDA(cudaMemcpyAsync(prm.edges, hb + H.edgeAt, (size_t)E * sizeof(RaEdge), cudaMemcpyHostToDevice, st));
  CS_CUDA(cudaMemcpyAsync(base + keysAt, hb + H.keysAt, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
  CS_CUDA(cudaMemcpyAsync(base + valsAt, hb + H.valsAt, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
  CS_CUDA(cub::DeviceRadixSort::SortPairs(base + tempAt, sortBytes, reinterpret_cast<int *>(base + keysAt),
                                          reinterpret_cast<int *>(base + keysSAt), reinterpret_cast<int *>(base + valsAt),
                                          reinterpret_cast<int *>(base + orderAt), n, 0, bits, st));
  void *args[] = {&prm};
  CS_CUDA(cudaLaunchCooperativeKernel((const void *)rotavg_kernel, dim3(wave), dim3(RA_THREADS), args, 0, st));
  count_launch();
  char *hw = c.h_rotavg.as<char>();
  CS_CUDA(cudaMemcpyAsync(hw, base + resAt, zeroEnd - resAt, cudaMemcpyDeviceToHost, st));
  CS_CUDA(cudaMemcpyAsync(hw + H.nodeAt, prm.nodes, (size_t)C * sizeof(RaNode), cudaMemcpyDeviceToHost, st));
  CS_CUDA(cudaMemcpyAsync(hw + H.thetaAt, prm.theta, (size_t)E * sizeof(double), cudaMemcpyDeviceToHost, st));
  return 0;
}

int rotavg_result(const DeviceCtx &c, int numImages, int numEdges, int maxIterations, double maxAngleDeg,
                  double *R_out, double *residuals, unsigned char *inlier, double cost[2], double *trace,
                  long long stats[6])
{
  const RaHost H(numImages, numEdges, maxIterations);
  const char *hb = c.h_rotavg.as<const char>();
  const RaResult *res = reinterpret_cast<const RaResult *>(hb);
  const RaNode *nodes = reinterpret_cast<const RaNode *>(hb + H.nodeAt);
  const RaEdge *eds = reinterpret_cast<const RaEdge *>(hb + H.edgeAt);
  const double *theta = reinterpret_cast<const double *>(hb + H.thetaAt);
  long long reached = 0, active = 0, inliers = 0;
  for (int a = 0; a < numImages; a++) {
    for (int k = 0; k < 9; k++) R_out[9 * (size_t)a + k] = nodes[a].reached ? nodes[a].R[k] : NAN;
    reached += nodes[a].reached;
  }
  for (int e = 0; e < numEdges; e++) {
    const double deg = eds[e].active ? theta[e] * (180.0 / CUDART_PI) : NAN;
    const bool in = deg < maxAngleDeg;
    if (residuals) residuals[e] = deg;
    if (inlier) inlier[e] = in;
    active += eds[e].active;
    inliers += in;
  }
  cost[0] = res->cost[0];
  cost[1] = res->cost[1];
  if (trace) memcpy(trace, hb + H.traceAt, (size_t)maxIterations * 3 * sizeof(double));
  if (stats) {
    stats[0] = active;
    stats[1] = reached - 1;
    stats[2] = reached;
    stats[3] = (long long)res->iters;
    stats[4] = (long long)res->cgIters;
    stats[5] = inliers;
  }
  return (int)res->iters;
}

}  // namespace cs
