// mesh.cu -- Poisson surface reconstruction of an oriented point cloud on a regular grid (cs_poisson_mesh): the splat
// as a gather over cell-sorted points, the right-hand side, one cooperative kernel for the multigrid-preconditioned CG
// solve and the iso-value, and marching tetrahedra with trimming as count-scan-write passes.  Every rule is stated in
// cudasift_b200.h at cs_poisson_mesh; tests/mesh_oracle.py restates them in float64.  cs_poisson_mesh_screened (screened
// Poisson with a Neumann boundary) shares every kernel but the right-hand side and the solve; its rules are stated at
// cs_poisson_mesh_screened and restated in tests/mesh_screened_oracle.py.  The two solve kernels share the V-cycle
// schedule (over two overloads of each level operation), the preconditioned CG loop (mgpcg, given each call's operator
// pass) and the trilinear field at a point; each keeps its own set-up, true residual, tau and status rule.
//
// Determinism: no floating-point atomics.  Integer atomics only where the result does not depend on their order (the
// bounding box as ordered-integer max, the cell histogram, the kept-vertex bit masks).  Every floating-point sum has a
// fixed order that depends on the grid size or the point count only: a node's splat runs over its cells in ascending
// index and each cell's points in sorted order; a total over nodes or points is coop.cuh's three-level total (tiles of
// CO_TREE_TILE items, groups of MT tile partials, then the group partials: co_tree_tiles, co_tree_groups,
// co_tree_total).  The vertex and triangle lists are counted lists (counted_list.cuh), and the box is a max of
// common.cuh's ordered float keys (float_key).
#include <cooperative_groups.h>
#include <cub/cub.cuh>

#include "common.cuh"
#include "coop.cuh"
#include "counted_list.cuh"

namespace cg = cooperative_groups;

namespace cs {

namespace {

constexpr int MT = 256;           // threads per CTA of every mesh kernel
constexpr int NU = 2;             // red-black sweep pairs before (and black-red pairs after) the coarse correction
constexpr int NU_COARSE = 8;      // the coarsest level (4 cells): 8 red-black pairs, then 8 black-red pairs
constexpr int LOCAL_N = 16;       // levels of at most 16 cells per axis run inside CTA 0, without grid barriers
constexpr int MAX_LEVELS = 8;     // 512 -> 4 cells

// The device words of a call, copied back after the synchronize.  info[7] is cs_poisson_mesh's info_out.
struct MeshResult {
  double info[7];                 // o_x, o_y, o_z, h, tau, mean density, true relative residual
  unsigned int boxLo[3], boxHi[3];// max of ~key(x) and of key(x) over the used points (ordered-integer floats)
  unsigned int used;
  unsigned int status;            // 0 ok, 1 no used point or zero extent, 2 tau <= 0, 3 not converged
  int iters;
  long long counts[4];            // vertices and triangles before trimming, vertices and triangles after
  double omega;                   // the screened call's effective point weight (its info_out[7])
};

struct MeshLevel {
  float *x, *f, *t;               // solution, right-hand side, residual scratch
  int n;                          // cells per axis: (n + 1)^3 nodes
};

struct MeshParams {
  MeshResult *res;
  int N, M;                       // cells per axis, nodes (N + 1)^3
  int numPoints;
  const float *xyz, *nrm, *inten; // inputs (inten may be null)
  double scale;
  // points
  int *keys, *keysS, *vals, *order;
  double *gs, *ns;                // sorted grid coordinates and unit normals [used][3]
  float *Is;                      // sorted intensities [used] (with inten)
  int *cellCount, *cellStart;     // [N^3 + 1]
  // nodes
  float *chi, *r, *b, *V0, *V1, *V2, *D, *S;   // z, p, q of the solve alias V0, V1, V2
  MeshLevel lv[MAX_LEVELS];
  int levels;
  double *tilePart, *groupPart;
  int maxIterations;
  double tol2, trim;
  // extraction
  unsigned int *keptMask;         // 7 bits per node (a byte each), packed 4 per word
  int *kstart;                    // first kept vertex of each node (aliases r)
  int *blockCounts, *blockOffsets;// [4][numBlocks]: vertices, triangles before trimming, triangles kept, vertices kept
  int numBlocks;
  float *vertices, *vertexIntensity;
  int *triangles;
  int maxVertices, maxTriangles;
};

// A level of the screened call's V-cycle: MeshLevel's arrays plus the diagonal of its screening operator.  The level
// operations have an overload for each of MeshLevel and NLevel; the V-cycle schedule over them is one template.
struct NLevel {
  float *x, *f, *t, *s;
  int n;
};

// The screened call's fields, a second kernel argument so that MeshParams keeps its layout (the Dirichlet kernels read
// it through the constant bank, and their code stays as it was).
struct ScreenParams {
  double alpha;                   // pointWeight
  double *u;                      // omega B_p^T x per sorted point [used]
  NLevel lv[MAX_LEVELS];          // lv[l].x, f, t alias MeshParams::lv[l]
};

__device__ __forceinline__ bool point_used(const MeshParams &p, int i, double nh[3])
{
  const float *x = p.xyz + 3 * (size_t)i, *n = p.nrm + 3 * (size_t)i;
  bool ok = isfinite(x[0]) && isfinite(x[1]) && isfinite(x[2]) && isfinite(n[0]) && isfinite(n[1]) && isfinite(n[2]);
  if (!ok) return false;
  const double a = n[0], b = n[1], c = n[2];
  const double len = sqrt(a * a + b * b + c * c);
  if (!(len > 0.0)) return false;
  nh[0] = a / len; nh[1] = b / len; nh[2] = c / len;
  return true;
}

// The grid of the used points' box (every thread computes the same values from the same words).
struct Grid {
  double o[3], h;
  bool ok;
};
__device__ __forceinline__ Grid mesh_grid(const MeshParams &p)
{
  const MeshResult &R = *p.res;
  Grid g;
  double lo[3], hi[3], E = 0.0;
  for (int a = 0; a < 3; a++) {
    lo[a] = key_float(~R.boxLo[a]);
    hi[a] = key_float(R.boxHi[a]);
    E = fmax(E, hi[a] - lo[a]);
  }
  const double L = fmax(p.scale, (double)p.N / (double)(p.N - 8)) * E;
  g.h = L / p.N;
  for (int a = 0; a < 3; a++) g.o[a] = (lo[a] + hi[a]) / 2.0 - L / 2.0;
  g.ok = R.used > 0 && E > 0.0;
  return g;
}

__device__ __forceinline__ void node_ijk(int idx, int n1, int &i, int &j, int &k)
{
  i = idx % n1;
  const int r = idx / n1;
  j = r % n1;
  k = r / n1;
}

// ---- multigrid level operations (tid / nth: the threads taking part; sync: their barrier) ---------------------------
// Each operation has two overloads: on a MeshLevel the Dirichlet call's (interior nodes only, diagonal 6), on an NLevel
// the screened call's (every node, its in-grid neighbours, diagonal deg + s).  The V-cycle schedule over them is one.
struct GridTeam {
  cg::grid_group g;
  int tid, nth;
  __device__ void sync() { g.sync(); }
};
struct CtaTeam {
  int tid, nth;
  __device__ void sync() { __syncthreads(); }
};

// (6 x - sum of the 6 neighbours) at interior node idx of a level with n1 nodes per axis, in float, neighbours in the
// order -x, +x, -y, +y, -z, +z.
__device__ __forceinline__ float nbr_sum(const float *x, int idx, int n1)
{
  const int s = n1 * n1;
  return ((((x[idx - 1] + x[idx + 1]) + x[idx - n1]) + x[idx + n1]) + x[idx - s]) + x[idx + s];
}

// The in-grid neighbours of node idx = (i, j, k) of a level with n cells in the order -x, +x, -y, +y, -z, +z (an absent
// one adds 0, so an interior node gets nbr_sum's value), in float; deg receives their count.
__device__ __forceinline__ float nbr_sum_nm(const float *x, int idx, int i, int j, int k, int n, float &deg)
{
  const int n1 = n + 1, s = n1 * n1;
  const float a = i > 0 ? x[idx - 1] : 0.0f, b = i < n ? x[idx + 1] : 0.0f;
  const float c = j > 0 ? x[idx - n1] : 0.0f, d = j < n ? x[idx + n1] : 0.0f;
  const float e = k > 0 ? x[idx - s] : 0.0f, f = k < n ? x[idx + s] : 0.0f;
  deg = (float)((i > 0) + (i < n) + (j > 0) + (j < n) + (k > 0) + (k < n));
  return ((((a + b) + c) + d) + e) + f;
}

// The same in float64 from the floats.
__device__ __forceinline__ double nbr_sum_nm_d(const float *x, int idx, int i, int j, int k, int n, double &deg)
{
  const int n1 = n + 1, s = n1 * n1;
  const double a = i > 0 ? x[idx - 1] : 0.0, b = i < n ? x[idx + 1] : 0.0;
  const double c = j > 0 ? x[idx - n1] : 0.0, d = j < n ? x[idx + n1] : 0.0;
  const double e = k > 0 ? x[idx - s] : 0.0, f = k < n ? x[idx + s] : 0.0;
  deg = (double)((i > 0) + (i < n) + (j > 0) + (j < n) + (k > 0) + (k < n));
  return ((((a + b) + c) + d) + e) + f;
}

// One Gauss-Seidel half-sweep over the interior nodes of one colour ((i + j + k) & 1): x = (f + neighbours) / 6.
template <class T>
__device__ void rb_sweep(const MeshLevel &L, int colour, T &team)
{
  const int n1 = L.n + 1, m = n1 * n1 * n1;
  for (int idx = team.tid; idx < m; idx += team.nth) {
    int i, j, k;
    node_ijk(idx, n1, i, j, k);
    if (((i + j + k) & 1) != colour || i == 0 || j == 0 || k == 0 || i == L.n || j == L.n || k == L.n) continue;
    L.x[idx] = (L.f[idx] + nbr_sum(L.x, idx, n1)) / 6.0f;
  }
}

// The same over every node of one colour: x = (f + in-grid neighbours) / (deg + s).
template <class T>
__device__ void rb_sweep(const NLevel &L, int colour, T &team)
{
  const int n1 = L.n + 1, m = n1 * n1 * n1;
  for (int idx = team.tid; idx < m; idx += team.nth) {
    int i, j, k;
    node_ijk(idx, n1, i, j, k);
    if (((i + j + k) & 1) != colour) continue;
    float deg;
    const float nb = nbr_sum_nm(L.x, idx, i, j, k, L.n, deg);
    L.x[idx] = (L.f[idx] + nb) / (deg + L.s[idx]);
  }
}

// t = f - A x on the interior, 0 on the boundary.
template <class T>
__device__ void residual(const MeshLevel &L, T &team)
{
  const int n1 = L.n + 1, m = n1 * n1 * n1;
  for (int idx = team.tid; idx < m; idx += team.nth) {
    int i, j, k;
    node_ijk(idx, n1, i, j, k);
    const bool bnd = i == 0 || j == 0 || k == 0 || i == L.n || j == L.n || k == L.n;
    L.t[idx] = bnd ? 0.0f : L.f[idx] - (6.0f * L.x[idx] - nbr_sum(L.x, idx, n1));
  }
}

// t = f - ((deg + s) x - in-grid neighbours) at every node.
template <class T>
__device__ void residual(const NLevel &L, T &team)
{
  const int n1 = L.n + 1, m = n1 * n1 * n1;
  for (int idx = team.tid; idx < m; idx += team.nth) {
    int i, j, k;
    node_ijk(idx, n1, i, j, k);
    float deg;
    const float nb = nbr_sum_nm(L.x, idx, i, j, k, L.n, deg);
    L.t[idx] = L.f[idx] - ((deg + L.s[idx]) * L.x[idx] - nb);
  }
}

// Coarse right-hand side fc = (1/2) P^T t at the coarse interior nodes (0 on the boundary); xc = 0 everywhere.  The 27
// fine nodes 2Q + d, d in {-1, 0, 1}^3 (dz outer, dx inner), weigh prod (1 - |d_a| / 2).
template <class T>
__device__ void restrict_to(const MeshLevel &F, const MeshLevel &C, T &team)
{
  const int n1 = C.n + 1, m = n1 * n1 * n1, f1 = F.n + 1;
  for (int idx = team.tid; idx < m; idx += team.nth) {
    int I, J, K;
    node_ijk(idx, n1, I, J, K);
    C.x[idx] = 0.0f;
    if (I == 0 || J == 0 || K == 0 || I == C.n || J == C.n || K == C.n) {
      C.f[idx] = 0.0f;
      continue;
    }
    float s = 0.0f;
    for (int dz = -1; dz <= 1; dz++)
      for (int dy = -1; dy <= 1; dy++)
        for (int dx = -1; dx <= 1; dx++) {
          const float w = (dx ? 0.5f : 1.0f) * (dy ? 0.5f : 1.0f) * (dz ? 0.5f : 1.0f);
          s = fmaf(w, F.t[((2 * K + dz) * f1 + 2 * J + dy) * f1 + 2 * I + dx], s);
        }
    C.f[idx] = 0.5f * s;
  }
}

// The same at every coarse node over its in-grid fine nodes.
template <class T>
__device__ void restrict_to(const NLevel &F, const NLevel &C, T &team)
{
  const int n1 = C.n + 1, m = n1 * n1 * n1, f1 = F.n + 1;
  for (int idx = team.tid; idx < m; idx += team.nth) {
    int I, J, K;
    node_ijk(idx, n1, I, J, K);
    C.x[idx] = 0.0f;
    float s = 0.0f;
    for (int dz = -1; dz <= 1; dz++)
      for (int dy = -1; dy <= 1; dy++)
        for (int dx = -1; dx <= 1; dx++) {
          const int fi = 2 * I + dx, fj = 2 * J + dy, fk = 2 * K + dz;
          if (fi < 0 || fj < 0 || fk < 0 || fi > F.n || fj > F.n || fk > F.n) continue;
          const float w = (dx ? 0.5f : 1.0f) * (dy ? 0.5f : 1.0f) * (dz ? 0.5f : 1.0f);
          s = fmaf(w, F.t[(fk * f1 + fj) * f1 + fi], s);
        }
    C.f[idx] = 0.5f * s;
  }
}

// x += P xc at the fine interior nodes: trilinear interpolation of the coarse nodes (odd coordinates take the two
// neighbours with 1/2 each; z outer, x inner).
template <class T>
__device__ void prolong_add(const MeshLevel &C, const MeshLevel &F, T &team)
{
  const int n1 = F.n + 1, m = n1 * n1 * n1, c1 = C.n + 1;
  for (int idx = team.tid; idx < m; idx += team.nth) {
    int i, j, k;
    node_ijk(idx, n1, i, j, k);
    if (i == 0 || j == 0 || k == 0 || i == F.n || j == F.n || k == F.n) continue;
    float s = 0.0f;
    for (int bz = 0; bz <= (k & 1); bz++)
      for (int by = 0; by <= (j & 1); by++)
        for (int bx = 0; bx <= (i & 1); bx++) {
          const float w = ((i & 1) ? 0.5f : 1.0f) * ((j & 1) ? 0.5f : 1.0f) * ((k & 1) ? 0.5f : 1.0f);
          s = fmaf(w, C.x[((k / 2 + bz) * c1 + j / 2 + by) * c1 + i / 2 + bx], s);
        }
    F.x[idx] += s;
  }
}

// The same at every fine node.
template <class T>
__device__ void prolong_add(const NLevel &C, const NLevel &F, T &team)
{
  const int n1 = F.n + 1, m = n1 * n1 * n1, c1 = C.n + 1;
  for (int idx = team.tid; idx < m; idx += team.nth) {
    int i, j, k;
    node_ijk(idx, n1, i, j, k);
    float s = 0.0f;
    for (int bz = 0; bz <= (k & 1); bz++)
      for (int by = 0; by <= (j & 1); by++)
        for (int bx = 0; bx <= (i & 1); bx++) {
          const float w = ((i & 1) ? 0.5f : 1.0f) * ((j & 1) ? 0.5f : 1.0f) * ((k & 1) ? 0.5f : 1.0f);
          s = fmaf(w, C.x[((k / 2 + bz) * c1 + j / 2 + by) * c1 + i / 2 + bx], s);
        }
    F.x[idx] += s;
  }
}

// ---- the V-cycle schedule, on MeshLevel or NLevel levels ------------------------------------------------------------
template <class Lv, class T>
__device__ void smooth_pairs(const Lv &L, int pairs, bool redFirst, T &team)
{
  for (int s = 0; s < pairs; s++) {
    rb_sweep(L, redFirst ? 0 : 1, team);
    team.sync();
    rb_sweep(L, redFirst ? 1 : 0, team);
    team.sync();
  }
}

template <class Lv, class T>
__device__ void v_down(const Lv *lv, int l, T &team)
{
  smooth_pairs(lv[l], NU, true, team);
  residual(lv[l], team);
  team.sync();
  restrict_to(lv[l], lv[l + 1], team);
  team.sync();
}

template <class Lv, class T>
__device__ void v_up(const Lv *lv, int l, T &team)
{
  prolong_add(lv[l + 1], lv[l], team);
  team.sync();
  smooth_pairs(lv[l], NU, false, team);
}

// One V-cycle from x = 0 on level 0 (lv[0].x zeroed, lv[0].f set): the levels of more than LOCAL_N cells with grid
// barriers, the rest inside CTA 0.
template <class Lv>
__device__ void v_cycle(const Lv *lv, int levels, GridTeam &grid)
{
  const int last = levels - 1;
  int lg = 0;
  while (lg < last && lv[lg].n > LOCAL_N) lg++;
  for (int l = 0; l < lg; l++) v_down(lv, l, grid);
  if (blockIdx.x == 0) {
    CtaTeam cta{(int)threadIdx.x, (int)blockDim.x};
    for (int l = lg; l < last; l++) v_down(lv, l, cta);
    smooth_pairs(lv[last], NU_COARSE, true, cta);
    smooth_pairs(lv[last], NU_COARSE, false, cta);
    for (int l = last - 1; l >= lg; l--) v_up(lv, l, cta);
  }
  grid.sync();
  for (int l = lg - 1; l >= 0; l--) v_up(lv, l, grid);
}

// ---- the solve ------------------------------------------------------------------------------------------------------
// The three-level total of the tile partials over n items (co_tree_groups, then co_tree_total, each after a grid
// barrier); every thread receives the K totals.
template <int K>
__device__ __forceinline__ void grid_total(const MeshParams &p, int n, GridTeam &grid, double (&out)[K])
{
  grid.sync();
  co_tree_groups<K, MT>(n, p.tilePart, p.groupPart);
  grid.sync();
  co_tree_total<K, MT>(n, p.groupPart, out);
}

__device__ __forceinline__ double grid_total(const MeshParams &p, int n, GridTeam &grid)
{
  double t[1];
  grid_total<1>(p, n, grid, t);
  return t[0];
}

// A field trilinear at grid coordinates g (tau, the mean density): add(w, node) for the corners of g's cell
// c = clamp(floor(g), 0, N - 1), z outer and x inner, w = prod (t_a or 1 - t_a) with t = g - c.  The caller keeps the
// sums, so one weight serves chi and D together.
template <class F>
__device__ __forceinline__ void trilinear(const double *g, int N, int n1, F &&add)
{
  int c[3];
  double t[3];
  for (int a = 0; a < 3; a++) {
    c[a] = min(max((int)floor(g[a]), 0), N - 1);
    t[a] = g[a] - c[a];
  }
  for (int bz = 0; bz < 2; bz++)
    for (int by = 0; by < 2; by++)
      for (int bx = 0; bx < 2; bx++) {
        const double w = (bx ? t[0] : 1.0 - t[0]) * (by ? t[1] : 1.0 - t[1]) * (bz ? t[2] : 1.0 - t[2]);
        add(w, ((c[2] + bz) * n1 + c[1] + by) * n1 + c[0] + bx);
      }
}

// CG for A chi = b from chi = 0, preconditioned by one V-cycle on the levels lv (z = B r), until r.r <= tol^2 b.b,
// after maxIterations iterations, or when p.A p is not positive; z, p and q are V0, V1 and V2.  The operator pass of an
// iteration is pre_ap(p) once p is complete, then q_i = ap(p, i), the float (A p)_i, in one tile pass with p.q.  Every
// total is a fixed-order one in float64; the vectors are floats, updated in float64.  Returns the iterations; bb and
// rr receive b.b and the last r.r; chi is complete on return.
template <class Lv, class Pre, class Ap>
__device__ __forceinline__ int mgpcg(const MeshParams &p, const Lv *lv, GridTeam &grid, Pre &&pre_ap, Ap &&ap,
                                     double &bb, double &rr)
{
  const int M = p.M;
  float *x = p.chi, *r = p.r, *b = p.b, *z = p.V0, *pp = p.V1, *q = p.V2;
  double rz = 0.0;
  co_tree_tiles<1, MT>(M, p.tilePart, [&](int i, double *v) {
    r[i] = b[i];
    z[i] = 0.0f;
    v[0] += (double)b[i] * (double)b[i];
  });
  bb = grid_total(p, M, grid);
  rr = bb;
  int k = 0;
  bool done = rr <= p.tol2 * bb;
  if (!done) {
    v_cycle(lv, p.levels, grid);
    co_tree_tiles<1, MT>(M, p.tilePart, [&](int i, double *v) {
      pp[i] = z[i];
      v[0] += (double)r[i] * (double)z[i];
    });
    rz = grid_total(p, M, grid);
  }
  while (!done) {
    grid.sync();                                       // p complete before pre_ap and A p read it
    pre_ap(pp);
    co_tree_tiles<1, MT>(M, p.tilePart, [&](int i, double *v) {
      const float a = ap(pp, i);
      q[i] = a;
      v[0] += (double)pp[i] * (double)a;
    });
    const double pq = grid_total(p, M, grid);
    if (!(pq > 0.0)) break;
    const double alpha = rz / pq;
    co_tree_tiles<1, MT>(M, p.tilePart, [&](int i, double *v) {
      x[i] = (float)((double)x[i] + alpha * (double)pp[i]);
      const float ri = (float)((double)r[i] - alpha * (double)q[i]);
      r[i] = ri;
      z[i] = 0.0f;
      v[0] += (double)ri * (double)ri;
    });
    rr = grid_total(p, M, grid);
    k++;
    if (rr <= p.tol2 * bb || k >= p.maxIterations) break;
    v_cycle(lv, p.levels, grid);
    co_tree_tiles<1, MT>(M, p.tilePart, [&](int i, double *v) { v[0] += (double)r[i] * (double)z[i]; });
    const double rzNew = grid_total(p, M, grid);
    const double beta = rzNew / rz;
    rz = rzNew;
    for (int i = grid.tid; i < M; i += grid.nth) pp[i] = (float)((double)z[i] + beta * (double)pp[i]);
  }
  grid.sync();
  return k;
}

// ---- kernels --------------------------------------------------------------------------------------------------------
// The used points' count and box.
__global__ void __launch_bounds__(MT) mesh_box_kernel(MeshParams p)
{
  __shared__ unsigned int s_lo[3], s_hi[3], s_used;
  if (threadIdx.x < 3) s_lo[threadIdx.x] = s_hi[threadIdx.x] = 0;
  if (threadIdx.x == 0) s_used = 0;
  __syncthreads();
  unsigned int lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0}, used = 0;
  for (int i = blockIdx.x * MT + threadIdx.x; i < p.numPoints; i += gridDim.x * MT) {
    double nh[3];
    if (!point_used(p, i, nh)) continue;
    used++;
    for (int a = 0; a < 3; a++) {
      const unsigned int k = float_key(p.xyz[3 * (size_t)i + a]);
      lo[a] = max(lo[a], ~k);
      hi[a] = max(hi[a], k);
    }
  }
  for (int a = 0; a < 3; a++) {
    atomicMax(&s_lo[a], lo[a]);
    atomicMax(&s_hi[a], hi[a]);
  }
  atomicAdd(&s_used, used);
  __syncthreads();
  if (threadIdx.x < 3) {
    atomicMax(&p.res->boxLo[threadIdx.x], s_lo[threadIdx.x]);
    atomicMax(&p.res->boxHi[threadIdx.x], s_hi[threadIdx.x]);
  }
  if (threadIdx.x == 0) atomicAdd(&p.res->used, s_used);
}

// The grid, the sort keys (the cell of a used point, N^3 for the others), the point indices and the cell histogram.
__global__ void __launch_bounds__(MT) mesh_keys_kernel(MeshParams p)
{
  const Grid g = mesh_grid(p);
  const int N = p.N;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    MeshResult &R = *p.res;
    R.status = g.ok ? 0u : 1u;
    for (int a = 0; a < 3; a++) R.info[a] = g.ok ? g.o[a] : 0.0;
    R.info[3] = g.ok ? g.h : 0.0;
  }
  for (int i = blockIdx.x * MT + threadIdx.x; i < p.numPoints; i += gridDim.x * MT) {
    double nh[3];
    int key = N * N * N;
    if (g.ok && point_used(p, i, nh)) {
      int c[3];
      for (int a = 0; a < 3; a++) {
        const double ga = ((double)p.xyz[3 * (size_t)i + a] - g.o[a]) / g.h;
        c[a] = min(max((int)floor(ga), 0), N - 1);
      }
      key = (c[2] * N + c[1]) * N + c[0];
      atomicAdd(&p.cellCount[key], 1);
    }
    p.keys[i] = key;
    p.vals[i] = i;
  }
}

// The used points in sorted order: grid coordinates, unit normals and intensities.
__global__ void __launch_bounds__(MT) mesh_points_kernel(MeshParams p)
{
  if (p.res->status != 0) return;
  const Grid g = mesh_grid(p);
  const int used = (int)p.res->used;
  for (int s = blockIdx.x * MT + threadIdx.x; s < used; s += gridDim.x * MT) {
    const int i = p.order[s];
    double nh[3];
    point_used(p, i, nh);
    for (int a = 0; a < 3; a++) {
      p.gs[3 * (size_t)s + a] = ((double)p.xyz[3 * (size_t)i + a] - g.o[a]) / g.h;
      p.ns[3 * (size_t)s + a] = nh[a];
    }
    if (p.inten) p.Is[s] = p.inten[i];
  }
}

// The splat as a gather: node q sums the points of its (up to) 8 cells, cells in ascending index, points in sorted
// order, weight prod (1 - |g_a - q_a|), in float64, rounded once.
__global__ void __launch_bounds__(MT) mesh_splat_kernel(MeshParams p)
{
  const int N = p.N, n1 = N + 1;
  const bool ok = p.res->status == 0;
  for (int idx = blockIdx.x * MT + threadIdx.x; idx < p.M; idx += gridDim.x * MT) {
    int i, j, k;
    node_ijk(idx, n1, i, j, k);
    double v0 = 0.0, v1 = 0.0, v2 = 0.0, d = 0.0, s = 0.0;
    for (int cz = k - 1; ok && cz <= k; cz++)
      for (int cy = j - 1; cy <= j; cy++)
        for (int cx = i - 1; cx <= i; cx++) {
          if (cx < 0 || cy < 0 || cz < 0 || cx >= N || cy >= N || cz >= N) continue;
          const int c = (cz * N + cy) * N + cx;
          for (int e = p.cellStart[c], end = p.cellStart[c + 1]; e < end; e++) {
            const double *g = p.gs + 3 * (size_t)e, *n = p.ns + 3 * (size_t)e;
            const double w = (1.0 - fabs(g[0] - i)) * (1.0 - fabs(g[1] - j)) * (1.0 - fabs(g[2] - k));
            v0 += w * n[0];
            v1 += w * n[1];
            v2 += w * n[2];
            d += w;
            if (p.S) s += w * (double)p.Is[e];
          }
        }
    p.V0[idx] = (float)v0;
    p.V1[idx] = (float)v1;
    p.V2[idx] = (float)v2;
    p.D[idx] = (float)d;
    if (p.S) p.S[idx] = (float)s;
  }
}

// b = (h / 2) sum_a (V_a(q + e_a) - V_a(q - e_a)) at the interior nodes in float64 from the floats, rounded once; 0 on
// the boundary.  chi = 0.
__global__ void __launch_bounds__(MT) mesh_rhs_kernel(MeshParams p)
{
  const int N = p.N, n1 = N + 1, s = n1 * n1;
  const double h = p.res->info[3];
  const bool ok = p.res->status == 0;
  for (int idx = blockIdx.x * MT + threadIdx.x; idx < p.M; idx += gridDim.x * MT) {
    int i, j, k;
    node_ijk(idx, n1, i, j, k);
    double b = 0.0;
    if (ok && i > 0 && j > 0 && k > 0 && i < N && j < N && k < N)
      b = h / 2.0 * ((((double)p.V0[idx + 1] - (double)p.V0[idx - 1]) + ((double)p.V1[idx + n1] - (double)p.V1[idx - n1])) +
                     ((double)p.V2[idx + s] - (double)p.V2[idx - s]));
    p.b[idx] = (float)b;
    p.chi[idx] = 0.0f;
  }
}

// CG preconditioned by one V-cycle, then the true residual, tau and the mean density; one resident wave.
__global__ void __launch_bounds__(MT) mesh_solve_kernel(MeshParams p)
{
  MeshResult &R = *p.res;
  if (R.status != 0) return;                           // every CTA reads the same word
  GridTeam grid{cg::this_grid(), (int)(blockIdx.x * MT + threadIdx.x), (int)(gridDim.x * MT)};
  const int N = p.N, n1 = N + 1, ss = n1 * n1, M = p.M;
  const float *x = p.chi, *b = p.b;
  auto interior = [&](int idx) {
    int i, j, k;
    node_ijk(idx, n1, i, j, k);
    return i > 0 && j > 0 && k > 0 && i < N && j < N && k < N;
  };
  double bb, rr;
  const int k = mgpcg(
      p, p.lv, grid, [](const float *) {},
      [&](const float *pp, int i) { return interior(i) ? 6.0f * pp[i] - nbr_sum(pp, i, n1) : 0.0f; }, bb, rr);
  // the true residual b - A chi, in float64 from the floats
  co_tree_tiles<1, MT>(M, p.tilePart, [&](int i, double *v) {
    if (!interior(i)) return;
    const double ax = 6.0 * (double)x[i] - (((((double)x[i - 1] + (double)x[i + 1]) + (double)x[i - n1]) +
                                             (double)x[i + n1]) + (double)x[i - ss]) - (double)x[i + ss];
    const double e = (double)b[i] - ax;
    v[0] += e * e;
  });
  const double rt = grid_total(p, M, grid);
  // tau and the mean density: chi and D trilinear at each used point's g, in sorted order
  const int used = (int)R.used;
  co_tree_tiles<2, MT>(used, p.tilePart, [&](int s, double *v) {
    double sc = 0.0, sd = 0.0;
    trilinear(p.gs + 3 * (size_t)s, N, n1, [&](double w, int node) {
      sc += w * (double)x[node];
      sd += w * (double)p.D[node];
    });
    v[0] += sc;
    v[1] += sd;
  });
  double td[2];
  grid_total<2>(p, used, grid, td);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const double tau = td[0] / used;
    R.info[4] = tau;
    R.info[5] = td[1] / used;
    R.info[6] = bb > 0.0 ? sqrt(rt / bb) : 0.0;
    R.iters = k;
    R.status = !(tau > 0.0) ? 2u : rr <= p.tol2 * bb ? 0u : 3u;
  }
}

// ---- screened Poisson with a Neumann boundary (cs_poisson_mesh_screened) ---------------------------------------------
// The trilinear weights B_p of a point at grid coordinates g, at the corners of its cell clamp(floor(g), 0, N - 1)
// (z outer, x inner) in the splat's form prod (1 - |g_a - q_a|); returns the first corner's node.
__device__ __forceinline__ int point_weights(const double *g, int N, double w[8])
{
  const int n1 = N + 1;
  int c[3];
  for (int a = 0; a < 3; a++) c[a] = min(max((int)floor(g[a]), 0), N - 1);
  for (int b = 0; b < 8; b++)
    w[b] = (1.0 - fabs(g[0] - (c[0] + (b & 1)))) * (1.0 - fabs(g[1] - (c[1] + ((b >> 1) & 1)))) *
           (1.0 - fabs(g[2] - (c[2] + ((b >> 2) & 1))));
  return (c[2] * n1 + c[1]) * n1 + c[0];
}

__device__ __forceinline__ int corner_offset(int b, int n1) { return (b & 1) + ((b >> 1) & 1) * n1 + (b >> 2) * n1 * n1; }

// u_s = omega B_s^T x (float64 from the floats) over the used points, in sorted order.
__device__ __forceinline__ void screen_points(const MeshParams &p, const ScreenParams &sc, const float *x, double omega,
                                              int used, GridTeam &grid)
{
  const int n1 = p.N + 1;
  for (int s = grid.tid; s < used; s += grid.nth) {
    double w[8];
    const int q0 = point_weights(p.gs + 3 * (size_t)s, p.N, w);
    double acc = 0.0;
    for (int b = 0; b < 8; b++) acc += w[b] * (double)x[q0 + corner_offset(b, n1)];
    sc.u[s] = omega * acc;
  }
}

// (S x)_q = sum B_s(q) u_s over the points of q's (up to 8) cells, cells in ascending index and points in sorted order
// (each row of 2 cells is one contiguous run of sorted points), in float64.
__device__ __forceinline__ double screen_gather(const MeshParams &p, const ScreenParams &sc, int i, int j, int k)
{
  const int N = p.N;
  double acc = 0.0;
  const int x0 = max(i - 1, 0), x1 = min(i, N - 1);
  for (int cz = max(k - 1, 0); cz <= min(k, N - 1); cz++)
    for (int cy = max(j - 1, 0); cy <= min(j, N - 1); cy++) {
      const int row = (cz * N + cy) * N;
      for (int e = p.cellStart[row + x0], end = p.cellStart[row + x1 + 1]; e < end; e++) {
        const double *g = p.gs + 3 * (size_t)e;
        acc += (1.0 - fabs(g[0] - i)) * (1.0 - fabs(g[1] - j)) * (1.0 - fabs(g[2] - k)) * sc.u[e];
      }
    }
  return acc;
}

// b = div of the edge field g(q -> q + e_a) = (h / 2)(V_a(q) + V_a(q + e_a)) over the in-grid edges at every node, in
// float64 from the floats, rounded once: per axis V_a(q + e_a) - V_a(q - e_a) with both neighbours (the Dirichlet
// call's central difference), V_a(q) + V_a(q + e_a) at a low face, -(V_a(q - e_a) + V_a(q)) at a high face, then
// (h / 2) ((x + y) + z).  chi = 0.
__global__ void __launch_bounds__(MT) mesh_rhs_neumann_kernel(MeshParams p)
{
  const int N = p.N, n1 = N + 1, s = n1 * n1;
  const double h = p.res->info[3];
  const bool ok = p.res->status == 0;
  const float *V[3] = {p.V0, p.V1, p.V2};
  for (int idx = blockIdx.x * MT + threadIdx.x; idx < p.M; idx += gridDim.x * MT) {
    int q[3];
    node_ijk(idx, n1, q[0], q[1], q[2]);
    double b = 0.0;
    if (ok) {
      double d[3];
      for (int a = 0; a < 3; a++) {
        const int st = a == 0 ? 1 : a == 1 ? n1 : s;
        const float *Va = V[a];
        d[a] = q[a] == 0   ? (double)Va[idx] + (double)Va[idx + st]
               : q[a] == N ? -((double)Va[idx - st] + (double)Va[idx])
                           : (double)Va[idx + st] - (double)Va[idx - st];
      }
      b = h / 2.0 * ((d[0] + d[1]) + d[2]);
    }
    p.b[idx] = (float)b;
    p.chi[idx] = 0.0f;
  }
}

// The screened solve: omega from the mean density, the levels' screening diagonals, CG on A = L + omega sum B B^T
// preconditioned by one V-cycle on L_l + diag(s_l), then the true residual, tau and the mean density; one resident
// wave.
__global__ void __launch_bounds__(MT) mesh_screened_solve_kernel(MeshParams p, ScreenParams sc)
{
  MeshResult &R = *p.res;
  if (R.status != 0) return;                           // every CTA reads the same word
  GridTeam grid{cg::this_grid(), (int)(blockIdx.x * MT + threadIdx.x), (int)(gridDim.x * MT)};
  const int N = p.N, n1 = N + 1, M = p.M, used = (int)R.used;
  const float *x = p.chi, *b = p.b;
  // F trilinear at sorted point s
  auto at_point = [&](const float *F, int s) {
    double acc = 0.0;
    trilinear(p.gs + 3 * (size_t)s, N, n1, [&](double w, int node) { acc += w * (double)F[node]; });
    return acc;
  };

  // omega = alpha / mean density
  co_tree_tiles<1, MT>(used, p.tilePart, [&](int s, double *v) { v[0] += at_point(p.D, s); });
  const double dsum = grid_total(p, used, grid);
  const double omega = sc.alpha / (dsum / used);
  // the screening diagonal of every level: s_l(Q) = (omega / 2^l) sum (B^l_p(Q))^2 at g / 2^l, over the fine cells of
  // Q's support in ascending index (rows of cells as contiguous runs of sorted points)
  // (level 0: a thread per node over its rows in order; coarser levels: a warp per node, lane j summing the rows
  // j, j + 32, ... in order, then vp_warp_sum's butterfly, lane 0's value)
  auto diag_rows = [&](int l, int idx, int lane, int step) {
    const int c1 = sc.lv[l].n + 1, f = 1 << l;
    const double inv = 1.0 / f;
    int I, J, K;
    node_ijk(idx, c1, I, J, K);
    const int x0 = max(f * (I - 1), 0), x1 = min(f * (I + 1), N) - 1;
    const int y0 = max(f * (J - 1), 0), ny = min(f * (J + 1), N) - y0;
    const int z0 = max(f * (K - 1), 0), nz = min(f * (K + 1), N) - z0;
    double acc = 0.0;
    for (int rw = lane; rw < ny * nz; rw += step) {
      const int row = ((z0 + rw / ny) * N + y0 + rw % ny) * N;
      for (int e = p.cellStart[row + x0], end = p.cellStart[row + x1 + 1]; e < end; e++) {
        const double *g = p.gs + 3 * (size_t)e;
        const double w = (1.0 - fabs(g[0] * inv - I)) * (1.0 - fabs(g[1] * inv - J)) * (1.0 - fabs(g[2] * inv - K));
        acc += w * w;
      }
    }
    return acc;
  };
  for (int t = grid.tid; t < M; t += grid.nth) sc.lv[0].s[t] = (float)(omega * diag_rows(0, t, 0, 1));
  {
    const int lane = threadIdx.x & 31, warp = grid.tid >> 5, warps = grid.nth >> 5;
    int coarse = 0;
    for (int l = 1; l < p.levels; l++) coarse += (sc.lv[l].n + 1) * (sc.lv[l].n + 1) * (sc.lv[l].n + 1);
    for (int t = warp; t < coarse; t += warps) {
      int l = 1, idx = t;
      while (idx >= (sc.lv[l].n + 1) * (sc.lv[l].n + 1) * (sc.lv[l].n + 1)) {
        idx -= (sc.lv[l].n + 1) * (sc.lv[l].n + 1) * (sc.lv[l].n + 1);
        l++;
      }
      double v[1] = {diag_rows(l, idx, lane, 32)};
      vp_warp_sum(v);
      if (lane == 0) sc.lv[l].s[idx] = (float)(omega / (1 << l) * v[0]);
    }
  }

  // (mgpcg's first total, b.b, is behind a grid barrier, which also completes the diagonals)
  double bb, rr;
  const int k = mgpcg(p, sc.lv, grid,
                      [&](const float *pp) {
                        screen_points(p, sc, pp, omega, used, grid);
                        grid.sync();
                      },
                      [&](const float *pp, int i) {
                        int a, bq, c;
                        node_ijk(i, n1, a, bq, c);
                        float deg;
                        const float nb = nbr_sum_nm(pp, i, a, bq, c, N, deg);
                        return (deg * pp[i] - nb) + (float)screen_gather(p, sc, a, bq, c);
                      },
                      bb, rr);
  // the true residual b - A chi, in float64 from the floats
  screen_points(p, sc, x, omega, used, grid);
  grid.sync();
  co_tree_tiles<1, MT>(M, p.tilePart, [&](int i, double *v) {
    int a, bq, c;
    node_ijk(i, n1, a, bq, c);
    double deg;
    const double nb = nbr_sum_nm_d(x, i, a, bq, c, N, deg);
    const double e = (double)b[i] - ((deg * (double)x[i] - nb) + screen_gather(p, sc, a, bq, c));
    v[0] += e * e;
  });
  const double rt = grid_total(p, M, grid);
  // tau: chi trilinear at the used points, in sorted order
  co_tree_tiles<1, MT>(used, p.tilePart, [&](int s, double *v) { v[0] += at_point(x, s); });
  const double tsum = grid_total(p, used, grid);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    R.info[4] = tsum / used;
    R.info[5] = dsum / used;
    R.info[6] = bb > 0.0 ? sqrt(rt / bb) : 0.0;
    R.omega = omega;
    R.iters = k;
    R.status = rr <= p.tol2 * bb ? 0u : 3u;
  }
}

// ---- extraction -----------------------------------------------------------------------------------------------------
// Lattice direction of corner bits (x 1, y 2, z 4) -> direction index: (1,0,0) 0, (0,1,0) 1, (0,0,1) 2, (1,1,0) 3,
// (1,0,1) 4, (0,1,1) 5, (1,1,1) 6.
__constant__ int c_dirOf[8] = {-1, 0, 1, 3, 2, 4, 5, 6};
__constant__ int c_dirBits[7] = {1, 2, 4, 3, 5, 6, 7};
// The axis permutations of the six tetrahedra of a cell, in lexicographic order.
__constant__ int c_perm[6][3] = {{0, 1, 2}, {0, 2, 1}, {1, 0, 2}, {1, 2, 0}, {2, 0, 1}, {2, 1, 0}};

struct Extract {
  const float *chi, *D;
  double tau;
  double thr;                     // trim x mean density
  int N;
  __device__ int node(int i, int j, int k) const { return (k * (N + 1) + j) * (N + 1) + i; }
  __device__ bool inside(int idx) const { return (double)chi[idx] >= tau; }
  // t of the edge from node q along direction bits db, in float64 from the floats
  __device__ double edge_t(int q, int db) const
  {
    const int n1_ = N + 1;
    const int qb = q + (db & 1) + ((db >> 1) & 1) * n1_ + ((db >> 2) & 1) * n1_ * n1_;
    const double a = chi[q], bv = chi[qb];
    return (tau - a) / (bv - a);
  }
  __device__ double lerp_at(const float *F, int q, int db, double t) const
  {
    const int n1_ = N + 1;
    const int qb = q + (db & 1) + ((db >> 1) & 1) * n1_ + ((db >> 2) & 1) * n1_ * n1_;
    const double a = F[q];
    return a + t * ((double)F[qb] - a);
  }
  // the crossing edges of node (i, j, k): bit d set when q + delta_d lies in the grid and differs in inside
  __device__ unsigned int cross_mask(int i, int j, int k) const
  {
    const int q = node(i, j, k);
    const bool in = inside(q);
    unsigned int m = 0;
    for (int d = 0; d < 7; d++) {
      const int db = c_dirBits[d];
      const int a = i + (db & 1), b = j + ((db >> 1) & 1), c = k + ((db >> 2) & 1);
      if (a > N || b > N || c > N) continue;
      if (inside(node(a, b, c)) != in) m |= 1u << d;
    }
    return m;
  }
};

// An edge of a tetrahedron as (lower node, direction index); corners are bit patterns of the cell (x 1, y 2, z 4).
struct EdgeRef {
  int node, dir;
};

__device__ __forceinline__ int det3(const int a[3], const int b[3], const int c[3])
{
  return a[0] * (b[1] * c[2] - b[2] * c[1]) - a[1] * (b[0] * c[2] - b[2] * c[0]) + a[2] * (b[0] * c[1] - b[1] * c[0]);
}

// The triangles of cell (i, j, k) (all coordinates < N), tetrahedron by tetrahedron in lexicographic permutation order,
// emit(tet, k, EdgeRef[3]) in order.  Orientation: with the edge midpoints m (in doubled corner coordinates) and a
// point ref on the outside side, det(m1 - m0, m2 - m0, ref - m0) > 0, else the last two are swapped.
template <class F>
__device__ void cell_triangles(const Extract &X, int i, int j, int k, F &&emit)
{
  bool in[8];
  for (int c = 0; c < 8; c++) in[c] = X.inside(X.node(i + (c & 1), j + ((c >> 1) & 1), k + ((c >> 2) & 1)));
  for (int t = 0; t < 6; t++) {
    int cor[4];
    cor[0] = 0;
    cor[1] = 1 << c_perm[t][0];
    cor[2] = cor[1] | (1 << c_perm[t][1]);
    cor[3] = 7;
    int ins[4], outs[4], ni = 0, no = 0;
    for (int v = 0; v < 4; v++) {
      if (in[cor[v]]) ins[ni++] = cor[v];
      else outs[no++] = cor[v];
    }
    if (ni == 0 || ni == 4) continue;
    auto edge = [&](int a, int b) {
      const int lo = a & b;                            // corners of a chain: the lower one is a subset of the other
      const int hi = a | b;
      EdgeRef e;
      e.node = X.node(i + (lo & 1), j + ((lo >> 1) & 1), k + ((lo >> 2) & 1));
      e.dir = c_dirOf[hi & ~lo];
      return e;
    };
    auto mid2 = [](int a, int b, int m[3]) {
      for (int ax = 0; ax < 3; ax++) m[ax] = ((a >> ax) & 1) + ((b >> ax) & 1);
    };
    // pairs (corner, corner) of up to 4 vertices in cycle order, and the reference point (doubled coordinates)
    int pa[4], pb[4], nv, ref[3];
    if (ni == 1 || ni == 3) {
      const int a = ni == 1 ? ins[0] : outs[0];
      const int *o = ni == 1 ? outs : ins;
      for (int v = 0; v < 3; v++) { pa[v] = a; pb[v] = o[v]; }
      nv = 3;
      const int r = ni == 1 ? outs[0] : a;
      for (int ax = 0; ax < 3; ax++) ref[ax] = 2 * ((r >> ax) & 1);
    } else {
      const int a = ins[0], b = ins[1], c = outs[0], d = outs[1];
      pa[0] = a; pb[0] = c;
      pa[1] = a; pb[1] = d;
      pa[2] = b; pb[2] = d;
      pa[3] = b; pb[3] = c;
      nv = 4;
      for (int ax = 0; ax < 3; ax++) ref[ax] = ((c >> ax) & 1) + ((d >> ax) & 1);
    }
    int m0[3], m1[3], m2[3], e1[3], e2[3], e3[3];
    mid2(pa[0], pb[0], m0);
    mid2(pa[1], pb[1], m1);
    mid2(pa[2], pb[2], m2);
    for (int ax = 0; ax < 3; ax++) {
      e1[ax] = m1[ax] - m0[ax];
      e2[ax] = m2[ax] - m0[ax];
      e3[ax] = ref[ax] - m0[ax];
    }
    if (det3(e1, e2, e3) < 0) {                        // reverse the cycle, keeping its first vertex
      if (nv == 3) {
        const int ta = pa[1], tb = pb[1];
        pa[1] = pa[2]; pb[1] = pb[2];
        pa[2] = ta; pb[2] = tb;
      } else {
        const int ta = pa[1], tb = pb[1];
        pa[1] = pa[3]; pb[1] = pb[3];
        pa[3] = ta; pb[3] = tb;
      }
    }
    EdgeRef v[4];
    for (int u = 0; u < nv; u++) v[u] = edge(pa[u], pb[u]);
    const EdgeRef t0[3] = {v[0], v[1], v[2]};
    emit(t, 0, t0);
    if (nv == 4) {
      const EdgeRef t1[3] = {v[0], v[2], v[3]};
      emit(t, 1, t1);
    }
  }
}

__device__ __forceinline__ Extract extract_of(const MeshParams &p)
{
  Extract X;
  X.chi = p.chi;
  X.D = p.D;
  X.tau = p.res->info[4];
  X.thr = p.trim * p.res->info[5];
  X.N = p.N;
  return X;
}

__device__ __forceinline__ bool mesh_extracts(const MeshResult &R) { return R.status == 0 || R.status == 3; }

__device__ __forceinline__ bool vertex_kept(const Extract &X, const EdgeRef &e)
{
  const int db = c_dirBits[e.dir];
  return !(X.lerp_at(X.D, e.node, db, X.edge_t(e.node, db)) < X.thr);
}

// Step 1 of counted list `which` (counted_list.cuh) into blockCounts[which][blockIdx.x].  This is counted_cta_count
// with the slot's address formed by thread 0 after the sum; handing counted_cta_count the slot's pointer forms it in
// every thread before the sum, which changes the code of mesh_count_kernel and mesh_kept_kernel (whose SASS
// tests/test_mesh_screened_cpu.py pins).
__device__ __forceinline__ void block_counts(const MeshParams &p, int which, int v)
{
  using BR = cub::BlockReduce<int, MT>;
  __shared__ typename BR::TempStorage tmp;
  const int s = BR(tmp).Sum(v);
  if (threadIdx.x == 0) p.blockCounts[(size_t)which * p.numBlocks + blockIdx.x] = s;
  __syncthreads();
}

// Per block of MT nodes: crossing edges, triangles before and after trimming; the kept triangles' vertices get their
// bit in keptMask.
__global__ void __launch_bounds__(MT) mesh_count_kernel(MeshParams p)
{
  const int idx = blockIdx.x * MT + threadIdx.x;
  int nv = 0, nt = 0, nk = 0;
  if (idx < p.M && mesh_extracts(*p.res)) {
    const Extract X = extract_of(p);
    int i, j, k;
    node_ijk(idx, p.N + 1, i, j, k);
    nv = __popc(X.cross_mask(i, j, k));
    if (i < p.N && j < p.N && k < p.N)
      cell_triangles(X, i, j, k, [&](int, int, const EdgeRef *e) {
        nt++;
        if (!(vertex_kept(X, e[0]) && vertex_kept(X, e[1]) && vertex_kept(X, e[2]))) return;
        nk++;
        for (int u = 0; u < 3; u++)
          atomicOr(&p.keptMask[e[u].node >> 2], 1u << (8 * (e[u].node & 3) + e[u].dir));
      });
  }
  block_counts(p, 0, nv);
  block_counts(p, 1, nt);
  block_counts(p, 2, nk);
}

__device__ __forceinline__ unsigned int kept_bits(const MeshParams &p, int node)
{
  return (p.keptMask[node >> 2] >> (8 * (node & 3))) & 0x7fu;
}

__global__ void __launch_bounds__(MT) mesh_kept_kernel(MeshParams p)
{
  const int idx = blockIdx.x * MT + threadIdx.x;
  block_counts(p, 3, idx < p.M ? __popc(kept_bits(p, idx)) : 0);
}

// The kept vertices in ascending edge id (node, then direction), and each node's first kept index; the last block
// records the four totals.
__global__ void __launch_bounds__(MT) mesh_vertices_kernel(MeshParams p)
{
  MeshResult &R = *p.res;
  const int nb = p.numBlocks;
  if (blockIdx.x == nb - 1 && threadIdx.x < 4) {
    const int w = threadIdx.x == 0 ? 0 : threadIdx.x == 1 ? 1 : threadIdx.x == 2 ? 3 : 2;   // counts[] order
    R.counts[threadIdx.x] = counted_total(p.blockOffsets, p.blockCounts, (size_t)w * nb + nb - 1);
  }
  const int idx = blockIdx.x * MT + threadIdx.x;
  const unsigned int m = idx < p.M ? kept_bits(p, idx) : 0u;
  const int first = p.blockOffsets[3 * (size_t)nb + blockIdx.x] + counted_position<MT>(__popc(m));
  if (idx >= p.M) return;
  p.kstart[idx] = first;
  if (!m) return;
  const Extract X = extract_of(p);
  const double *o = R.info;
  const double h = R.info[3];
  int i, j, k;
  node_ijk(idx, p.N + 1, i, j, k);
  int v = first;
  for (int d = 0; d < 7; d++) {
    if (!((m >> d) & 1)) continue;
    if (v < p.maxVertices) {
      const int db = c_dirBits[d];
      const double t = X.edge_t(idx, db);
      const int q[3] = {i, j, k};
      for (int a = 0; a < 3; a++) p.vertices[3 * (size_t)v + a] = (float)(o[a] + h * (q[a] + t * ((db >> a) & 1)));
      if (p.vertexIntensity) {
        const double den = X.lerp_at(p.D, idx, db, t);
        p.vertexIntensity[v] = den != 0.0 ? (float)(X.lerp_at(p.S, idx, db, t) / den) : 0.0f;
      }
    }
    v++;
  }
}

// The kept triangles in ascending (cell, tetrahedron, k), their vertices as kept-vertex indices.
__global__ void __launch_bounds__(MT) mesh_triangles_kernel(MeshParams p)
{
  const int idx = blockIdx.x * MT + threadIdx.x;
  const Extract X = extract_of(p);
  int i = 0, j = 0, k = 0, nk = 0;
  if (idx < p.M) node_ijk(idx, p.N + 1, i, j, k);
  const bool cell = idx < p.M && mesh_extracts(*p.res) && i < p.N && j < p.N && k < p.N;
  auto each = [&](auto &&f) {
    cell_triangles(X, i, j, k, [&](int, int, const EdgeRef *e) {
      if (vertex_kept(X, e[0]) && vertex_kept(X, e[1]) && vertex_kept(X, e[2])) f(e);
    });
  };
  if (cell) each([&](const EdgeRef *) { nk++; });
  int t = p.blockOffsets[2 * (size_t)p.numBlocks + blockIdx.x] + counted_position<MT>(nk);
  if (!cell || !nk) return;
  each([&](const EdgeRef *e) {
    if (t < p.maxTriangles)
      for (int u = 0; u < 3; u++)
        p.triangles[3 * (size_t)t + u] =
            p.kstart[e[u].node] + __popc(kept_bits(p, e[u].node) & ((1u << e[u].dir) - 1u));
    t++;
  });
}

}  // namespace

// Bytes of (n + 1)^3 floats.
static size_t level_bytes(int n) { return (size_t)(n + 1) * (n + 1) * (n + 1) * sizeof(float); }

int mesh_run(const float *xyz, const float *normal, const float *intensity, int numPoints, int depth, double scale,
             double pointWeight, int maxIterations, double tol, double trim, float *vertices, float *vertexIntensity,
             int maxVertices, int *triangles, int maxTriangles, float *chiOut, cudaStream_t st, void *h_result)
{
  const bool screened = pointWeight > 0.0;
  const int N = 1 << depth, n1 = N + 1;
  const int M = n1 * n1 * n1;
  const int P = numPoints;
  const bool hasI = intensity != nullptr;
  const int nb = idivup(M, MT);
  const int tilesMax = std::max(idivup(M, CO_TREE_TILE), idivup(std::max(P, 1), CO_TREE_TILE));
  const int groupsMax = idivup(tilesMax, MT);          // a group is MT tile partials
  const int bits = radix_bits((long long)N * N * N);

  size_t sortBytes = 0, scanBytes = 0, scanBytes2 = 0;
  CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sortBytes, (int *)nullptr, (int *)nullptr, (int *)nullptr,
                                          (int *)nullptr, std::max(P, 1), 0, bits, st));
  CS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scanBytes, (int *)nullptr, (int *)nullptr, N * N * N + 1, st));
  CS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scanBytes2, (int *)nullptr, (int *)nullptr, nb, st));
  Layout L(256);
  const size_t resAt = L.take(sizeof(MeshResult));
  const size_t maskAt = L.take((size_t)idivup(M, 4) * sizeof(unsigned int));
  const size_t zeroEnd = L.bytes;
  const size_t chiAt = L.take(level_bytes(N)), rAt = L.take(level_bytes(N)), bAt = L.take(level_bytes(N));
  const size_t v0At = L.take(level_bytes(N)), v1At = L.take(level_bytes(N)), v2At = L.take(level_bytes(N));
  const size_t dAt = L.take(level_bytes(N)), sAt = hasI ? L.take(level_bytes(N)) : 0;
  size_t lvAt[MAX_LEVELS][3];
  int levels = 1;
  for (int n = N / 2; n >= 4; n /= 2, levels++)
    for (int a = 0; a < 3; a++) lvAt[levels][a] = L.take(level_bytes(n));
  const size_t keysAt = L.take((size_t)P * sizeof(int)), keysSAt = L.take((size_t)P * sizeof(int));
  const size_t valsAt = L.take((size_t)P * sizeof(int)), orderAt = L.take((size_t)P * sizeof(int));
  const size_t gsAt = L.take((size_t)P * 3 * sizeof(double)), nsAt = L.take((size_t)P * 3 * sizeof(double));
  const size_t isAt = hasI ? L.take((size_t)P * sizeof(float)) : 0;
  const size_t tileAt = L.take((size_t)tilesMax * 2 * sizeof(double));
  const size_t groupAt = L.take((size_t)groupsMax * 2 * sizeof(double));
  const size_t cntAt = L.take((size_t)4 * nb * sizeof(int)), offAt = L.take((size_t)4 * nb * sizeof(int));
  const size_t tempAt = L.take(std::max(sortBytes, std::max(scanBytes, scanBytes2)));
  // the screened call: the levels' screening diagonals, u, and cell starts of their own (the solve reads them)
  size_t diagAt[MAX_LEVELS] = {}, uAt = 0, startAt = 0;
  if (screened) {
    for (int l = 0, n = N; l < levels; l++, n /= 2) diagAt[l] = L.take(level_bytes(n));
    uAt = L.take((size_t)P * sizeof(double));
    startAt = L.take(((size_t)N * N * N + 1) * sizeof(int));
  }

  char *base = nullptr;
  CS_CUDA(cudaMallocAsync((void **)&base, L.bytes, st));
  auto at = [&](size_t off) { return base + off; };

  MeshParams p{};
  p.res = reinterpret_cast<MeshResult *>(at(resAt));
  p.N = N;
  p.M = M;
  p.numPoints = P;
  p.xyz = xyz;
  p.nrm = normal;
  p.inten = intensity;
  p.scale = scale;
  p.keys = reinterpret_cast<int *>(at(keysAt));
  p.keysS = reinterpret_cast<int *>(at(keysSAt));
  p.vals = reinterpret_cast<int *>(at(valsAt));
  p.order = reinterpret_cast<int *>(at(orderAt));
  p.gs = reinterpret_cast<double *>(at(gsAt));
  p.ns = reinterpret_cast<double *>(at(nsAt));
  p.Is = hasI ? reinterpret_cast<float *>(at(isAt)) : nullptr;
  p.chi = reinterpret_cast<float *>(at(chiAt));
  p.r = reinterpret_cast<float *>(at(rAt));
  p.b = reinterpret_cast<float *>(at(bAt));
  p.V0 = reinterpret_cast<float *>(at(v0At));
  p.V1 = reinterpret_cast<float *>(at(v1At));
  p.V2 = reinterpret_cast<float *>(at(v2At));
  p.D = reinterpret_cast<float *>(at(dAt));
  p.S = hasI ? reinterpret_cast<float *>(at(sAt)) : nullptr;
  p.cellCount = reinterpret_cast<int *>(p.chi);        // dead before the right-hand side zeroes chi
  p.cellStart = reinterpret_cast<int *>(screened ? at(startAt) : at(rAt));   // Dirichlet: dead before the solve writes r
  p.kstart = reinterpret_cast<int *>(p.r);             // r is dead after the solve
  p.lv[0] = MeshLevel{p.V0, p.r, p.V2, N};             // z = M r, with q as the residual scratch
  for (int l = 1, n = N / 2; l < levels; l++, n /= 2)
    p.lv[l] = MeshLevel{reinterpret_cast<float *>(at(lvAt[l][0])), reinterpret_cast<float *>(at(lvAt[l][1])),
                        reinterpret_cast<float *>(at(lvAt[l][2])), n};
  p.levels = levels;
  p.tilePart = reinterpret_cast<double *>(at(tileAt));
  p.groupPart = reinterpret_cast<double *>(at(groupAt));
  p.maxIterations = maxIterations;
  p.tol2 = tol * tol;
  p.trim = trim;
  p.keptMask = reinterpret_cast<unsigned int *>(at(maskAt));
  p.blockCounts = reinterpret_cast<int *>(at(cntAt));
  p.blockOffsets = reinterpret_cast<int *>(at(offAt));
  p.numBlocks = nb;
  p.vertices = vertices;
  p.vertexIntensity = vertexIntensity;
  p.triangles = triangles;
  p.maxVertices = maxVertices;
  p.maxTriangles = maxTriangles;
  void *temp = at(tempAt);
  ScreenParams sc{};
  sc.alpha = pointWeight;
  if (screened) {
    sc.u = reinterpret_cast<double *>(at(uAt));
    for (int l = 0; l < levels; l++)
      sc.lv[l] = NLevel{p.lv[l].x, p.lv[l].f, p.lv[l].t, reinterpret_cast<float *>(at(diagAt[l])), p.lv[l].n};
  }

  const int wave = screened ? coop_grid<mesh_screened_solve_kernel, MT>("cs_poisson_mesh_screened")
                            : coop_grid<mesh_solve_kernel, MT>("cs_poisson_mesh");
  int r = wave < 0 ? wave : 0;
  cudaEvent_t *tev = match_timing_events();
  const int pointCtas = std::max(1, std::min(idivup(P, MT), 4096));
  const int nodeCtas = std::min(nb, 65536);
  auto launch = [&]() -> int {
    if (r < 0) return r;
    if (tev) CS_CUDA(cudaEventRecord(tev[0], st));
    CS_CUDA(cudaMemsetAsync(base, 0, zeroEnd, st));
    CS_CUDA(cudaMemsetAsync(p.cellCount, 0, ((size_t)N * N * N + 1) * sizeof(int), st));
    mesh_box_kernel<<<pointCtas, MT, 0, st>>>(p);
    mesh_keys_kernel<<<pointCtas, MT, 0, st>>>(p);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    CS_CUDA(cub::DeviceRadixSort::SortPairs(temp, sortBytes, p.keys, p.keysS, p.vals, p.order, P, 0, bits, st));
    CS_CUDA(cub::DeviceScan::ExclusiveSum(temp, scanBytes, p.cellCount, p.cellStart, N * N * N + 1, st));
    mesh_points_kernel<<<pointCtas, MT, 0, st>>>(p);
    mesh_splat_kernel<<<nodeCtas, MT, 0, st>>>(p);
    if (screened) mesh_rhs_neumann_kernel<<<nodeCtas, MT, 0, st>>>(p);
    else mesh_rhs_kernel<<<nodeCtas, MT, 0, st>>>(p);
    count_launch(3);
    CS_CUDA(cudaGetLastError());
    if (tev) CS_CUDA(cudaEventRecord(tev[1], st));
    void *args[] = {&p, &sc};
    if (screened)
      CS_CUDA(cudaLaunchCooperativeKernel((const void *)mesh_screened_solve_kernel, dim3(wave), dim3(MT), args, 0, st));
    else
      CS_CUDA(cudaLaunchCooperativeKernel((const void *)mesh_solve_kernel, dim3(wave), dim3(MT), args, 0, st));
    count_launch();
    if (tev) CS_CUDA(cudaEventRecord(tev[2], st));
    mesh_count_kernel<<<nb, MT, 0, st>>>(p);
    mesh_kept_kernel<<<nb, MT, 0, st>>>(p);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    for (int w = 0; w < 4; w++)
      CS_CUDA(cub::DeviceScan::ExclusiveSum(temp, scanBytes2, p.blockCounts + (size_t)w * nb,
                                            p.blockOffsets + (size_t)w * nb, nb, st));
    mesh_vertices_kernel<<<nb, MT, 0, st>>>(p);
    mesh_triangles_kernel<<<nb, MT, 0, st>>>(p);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    if (tev) CS_CUDA(cudaEventRecord(tev[3], st));
    if (chiOut) CS_CUDA(cudaMemcpyAsync(chiOut, p.chi, level_bytes(N), cudaMemcpyDeviceToDevice, st));
    CS_CUDA(cudaMemcpyAsync(h_result, p.res, sizeof(MeshResult), cudaMemcpyDeviceToHost, st));
    if (tev) {
      static const char *const names[3] = {"splat", "solve", "extract"};
      report_stage_times(tev, names, 3, "mesh timing depth=%d points=%d%s", depth, P, screened ? " screened" : "");
    }
    return 0;
  };
  r = launch();
  cudaFreeAsync(base, st);
  return r;
}

size_t mesh_result_bytes() { return sizeof(MeshResult); }

// stats_out and info_out from the result words (after the synchronize); returns the full triangle count.
int mesh_result(const void *h_result, int numPoints, int maxVertices, int maxTriangles, bool screened, double *info,
                long long stats[10])
{
  const MeshResult &R = *static_cast<const MeshResult *>(h_result);
  if (info) {
    for (int k = 0; k < 7; k++) info[k] = R.info[k];
    if (screened) info[7] = R.omega;
  }
  const bool out = R.status == 0 || R.status == 3;
  const long long c[4] = {out ? R.counts[0] : 0, out ? R.counts[1] : 0, out ? R.counts[2] : 0, out ? R.counts[3] : 0};
  if (stats) {
    stats[0] = R.used;
    stats[1] = numPoints - (long long)R.used;
    stats[2] = R.status == 1 ? 0 : R.iters;
    stats[3] = c[0];
    stats[4] = c[1];
    stats[5] = c[2];
    stats[6] = c[3];
    stats[7] = std::min(c[2], (long long)maxVertices);
    stats[8] = std::min(c[3], (long long)maxTriangles);
    stats[9] = R.status;
  }
  return (int)c[3];
}

}  // namespace cs
