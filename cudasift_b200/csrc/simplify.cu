// simplify.cu -- quadric-error edge collapse (cs_simplify_mesh) in independent parallel passes: the vertex -> face
// adjacency by a stable sort of corner keys, one thread per edge for the validity tests, position and cost, a radix
// sort of the candidate keys for the gating threshold, an atomicMin scatter of keys onto the closed 1-rings of both
// ends and the selection test, the collapse, and the face remap as count-scan-write passes (the faces and the output
// vertices are counted lists of counted_list.cuh).  The float64 vectors, the tie order s(id), the input check and the
// launch shape are shared with texture.cu in trimesh.cuh.  Every rule is stated in cudasift_b200.h at
// cs_simplify_mesh; tests/simplify_oracle.py restates them in float64.
//
// Determinism: no floating-point atomics; integer atomics only where the result does not depend on their order (counts,
// the minimum key of a vertex, the largest applied error as ordered bits).  This unit is compiled with -fmad=false so
// that every float64 product and sum is rounded once, in the order written, as the oracle computes it.
#include <math_constants.h>

#include <cmath>
#include <cstring>

#include <cub/cub.cuh>

#include "common.cuh"
#include "counted_list.cuh"
#include "trimesh.cuh"

namespace cs {

namespace {

constexpr int F_SHIFT = 1;                    // f = 1/2: the cheapest ceil(C / 2) candidates compete in a pass
constexpr double DET_EPS = 1e-6;              // the minimiser is used when det(A) > DET_EPS a11 a22 a33
constexpr int MAX_PASSES = 1000;
constexpr unsigned long long NO_KEY = ~0ull;

// The device words of a call, copied back after each pass.
struct SimplifyResult {
  unsigned int bad;                           // an invalid input (status 2)
  unsigned int frozen;                        // frozen vertices
  unsigned int cand, sel, drops;              // this pass: candidates, selected edges, their faces
  unsigned int applied;                       // the target pass: edges applied
  unsigned int tris;                          // the target pass: triangles left
  unsigned int verts;                         // output vertices
  unsigned long long maxErr;                  // the largest applied cost / A (its float64 bits)
  unsigned long long thr, cut;                // gating threshold, the target pass's last applied key
};

struct SimplifyParams {
  SimplifyResult *res;
  int V, T;                                   // vertices, current triangles
  const float *vin, *iin;                     // input vertices [V][3], intensities [V] (or null)
  const int *tin;                             // input triangles [T0][3]
  int *tri, *triN, *tid, *tidN;               // current and next triangles and their input indices
  int *ckey, *ckeyS, *cval, *cvalS;           // corner keys (vertex) and values (corner), sorted
  int *vcount, *vstart;                       // faces per vertex, the exclusive scan [V + 1]
  double *pos, *Q, *A;                        // [V][3], [V][10], [V]
  float *inten;                               // [V] (or null)
  unsigned char *frozen;
  int *remap, *used;
  unsigned long long *key, *keyS, *mark, *selKey, *selKeyS;
  int *drops, *dropsS, *cum;
  int *blockCounts, *blockOffsets;
  double bw, maxError;
  float *outV, *outI;
  int *outT;
  int maxOutV, maxOutT;
};

// q += w p p^T for the plane (n, d): the upper triangle row-major, each entry w (p_i p_j)
__device__ void plane_add(double *q, D3 n, double d, double w)
{
  const double pl[4] = {n.x, n.y, n.z, d};
  int k = 0;
  for (int i = 0; i < 4; i++)
    for (int j = i; j < 4; j++, k++) q[k] = q[k] + w * (pl[i] * pl[j]);
}

__device__ double cost_of(const double *q, D3 x)
{
  const double a11 = q[0], a12 = q[1], a13 = q[2], b1 = q[3], a22 = q[4], a23 = q[5], b2 = q[6], a33 = q[7],
               b3 = q[8], c = q[9];
  double r = (a11 * x.x * x.x + a22 * x.y * x.y) + a33 * x.z * x.z;
  r = r + 2.0 * ((a12 * x.x * x.y + a13 * x.x * x.z) + a23 * x.y * x.z);
  r = r + 2.0 * ((b1 * x.x + b2 * x.y) + b3 * x.z);
  return r + c;
}

__device__ double optimum(const double *q, D3 pu, D3 pv, D3 &x)
{
  const double a11 = q[0], a12 = q[1], a13 = q[2], b1 = q[3], a22 = q[4], a23 = q[5], b2 = q[6], a33 = q[7],
               b3 = q[8];
  const double c11 = a22 * a33 - a23 * a23, c12 = a12 * a33 - a23 * a13, c13 = a12 * a23 - a22 * a13;
  const double det = (a11 * c11 - a12 * c12) + a13 * c13;
  double best;
  if (det > DET_EPS * (a11 * a22 * a33)) {
    x.x = -(((b1 * c11 - a12 * (b2 * a33 - a23 * b3)) + a13 * (b2 * a23 - a22 * b3)) / det);
    x.y = -(((a11 * (b2 * a33 - a23 * b3) - b1 * c12) + a13 * (a12 * b3 - b2 * a13)) / det);
    x.z = -(((a11 * (a22 * b3 - b2 * a23) - a12 * (a12 * b3 - b2 * a13)) + b1 * c13) / det);
    best = cost_of(q, x);
  } else {
    x = pu;
    best = cost_of(q, pu);
    const double cv = cost_of(q, pv);
    if (cv < best) { x = pv; best = cv; }
    const D3 mid = {(pu.x + pv.x) * 0.5, (pu.y + pv.y) * 0.5, (pu.z + pv.z) * 0.5};
    const double cm = cost_of(q, mid);
    if (cm < best) { x = mid; best = cm; }
  }
  return best > 0.0 ? best : 0.0;
}

// The faces of x: sorted corners vstart[x] .. vstart[x + 1], face c / 3 at position c % 3, ascending.
template <class F>
__device__ __forceinline__ bool any_face(const SimplifyParams &p, int x, F &&f)
{
  for (int i = p.vstart[x], e = p.vstart[x + 1]; i < e; i++) {
    const int c = p.cvalS[i], t = c / 3;
    if (f(t, c - 3 * t)) return true;
  }
  return false;
}

__device__ __forceinline__ int corner(const SimplifyParams &p, int t, int j) { return p.tri[3 * t + j % 3]; }

// some face of x traverses a -> b
__device__ bool has_directed(const SimplifyParams &p, int x, int a, int b)
{
  return any_face(p, x, [&](int t, int) {
    for (int j = 0; j < 3; j++)
      if (corner(p, t, j) == a && corner(p, t, j + 1) == b) return true;
    return false;
  });
}

__device__ bool face_has(const SimplifyParams &p, int t, int w)
{
  return corner(p, t, 0) == w || corner(p, t, 1) == w || corner(p, t, 2) == w;
}

__device__ bool on_boundary(const SimplifyParams &p, int x)
{
  return any_face(p, x, [&](int t, int j) { return !has_directed(p, x, corner(p, t, j + 1), x); });
}

__device__ bool boundary_edge(const SimplifyParams &p, int x, int y)
{
  return !(has_directed(p, x, x, y) && has_directed(p, x, y, x));
}

// The edge at corner k of face t (rules 3 and 4): false when it is not the canonical corner or its collapse is not
// valid or not admissible; else u < v, the position x, the error cost / A and the faces it drops.
__device__ bool evaluate(const SimplifyParams &p, int t, int k, int &u, int &v, D3 &x, double &err, int &drops)
{
  const int a = corner(p, t, k), b = corner(p, t, k + 1);
  if (p.frozen[a] || p.frozen[b]) return false;
  const bool interior = has_directed(p, b, b, a);
  if (interior && !(a < b)) return false;
  u = min(a, b);
  v = max(a, b);
  const int w1 = corner(p, t, k + 2);
  int w2 = -1;
  if (interior)
    any_face(p, b, [&](int s, int j) {
      if (corner(p, s, j + 1) != a) return false;
      w2 = corner(p, s, j + 2);
      return true;
    });
  // link condition: every common neighbour is an apex of a face on uv
  const int uu = u, vv = v;
  if (any_face(p, uu, [&](int s, int) {
        for (int j = 0; j < 3; j++) {
          const int w = corner(p, s, j);
          if (w == uu || w == vv || w == w1 || w == w2) continue;
          if (any_face(p, vv, [&](int r, int) { return face_has(p, r, w); })) return true;
        }
        return false;
      }))
    return false;
  if (interior) {
    if (on_boundary(p, u) && on_boundary(p, v)) return false;
    auto both = [&](int s, int) { return face_has(p, s, w1) && face_has(p, s, w2); };
    if (any_face(p, uu, both) && any_face(p, vv, both)) return false;
  } else if (boundary_edge(p, u, w1) && boundary_edge(p, v, w1)) {
    return false;
  }
  double q[10];
  for (int i = 0; i < 10; i++) q[i] = p.Q[10 * (size_t)u + i] + p.Q[10 * (size_t)v + i];
  const double area = p.A[u] + p.A[v];
  const D3 pu = vertex_of(p.pos, u), pv = vertex_of(p.pos, v);
  const double cst = optimum(q, pu, pv, x);
  err = area > 0.0 ? cst / area : (cst == 0.0 ? 0.0 : CUDART_INF);
  if (!(err < CUDART_INF && sqrt(err) <= p.maxError)) return false;
  // flips: every face of u, then of v, without both
  const D3 xx = x;
  auto flips = [&](int s, int) {
    const int g0 = corner(p, s, 0), g1 = corner(p, s, 1), g2 = corner(p, s, 2);
    const bool hu = g0 == uu || g1 == uu || g2 == uu, hv = g0 == vv || g1 == vv || g2 == vv;
    if (hu && hv) return false;
    const D3 p0 = vertex_of(p.pos, g0), p1 = vertex_of(p.pos, g1), p2 = vertex_of(p.pos, g2);
    const D3 n0 = normal3(p0, p1, p2);
    if (!(dot3(n0, n0) > 0.0)) return false;
    auto moved = [&](int g, D3 q0) { return (g == uu || g == vv) ? xx : q0; };
    return !(dot3(n0, normal3(moved(g0, p0), moved(g1, p1), moved(g2, p2))) > 0.0);
  };
  if (any_face(p, uu, flips) || any_face(p, vv, flips)) return false;
  drops = interior ? 2 : 1;
  return true;
}

// ---- setup ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MT) simplify_init_kernel(SimplifyParams p)
{
  const int n = max(p.V, p.T);
  for (int i = blockIdx.x * MT + threadIdx.x; i < n; i += gridDim.x * MT) {
    if (i < p.V) {
      for (int d = 0; d < 3; d++) p.pos[3 * (size_t)i + d] = (double)p.vin[3 * (size_t)i + d];
      if (p.inten) p.inten[i] = p.iin[i];
      p.remap[i] = i;
    }
    if (i < p.T) {
      for (int d = 0; d < 3; d++) p.tri[3 * (size_t)i + d] = p.tin[3 * (size_t)i + d];
      p.tid[i] = i;
    }
  }
}

// corner keys and the faces per vertex (cub's stable radix sort then orders each vertex's faces by index)
__global__ void __launch_bounds__(MT) simplify_corners_kernel(SimplifyParams p)
{
  for (int c = blockIdx.x * MT + threadIdx.x; c < 3 * p.T; c += gridDim.x * MT) {
    const int x = p.tri[c];
    p.ckey[c] = x;
    p.cval[c] = c;
    atomicAdd(&p.vcount[x], 1);
  }
}

// frozen status and the quadric of every vertex with faces (rules 1 and 2)
__global__ void __launch_bounds__(MT) simplify_vertex_kernel(SimplifyParams p)
{
  const int x = blockIdx.x * MT + threadIdx.x;
  if (x >= p.V) return;
  const int s0 = p.vstart[x], k = p.vstart[x + 1] - s0;
  double *q = p.Q + 10 * (size_t)x;
  for (int i = 0; i < 10; i++) q[i] = 0.0;
  p.A[x] = 0.0;
  p.frozen[x] = 0;
  if (k == 0) return;
  auto face = [&](int i) { return p.cvalS[s0 + i] / 3; };
  auto at = [&](int i) { return p.cvalS[s0 + i] % 3; };
  auto nxt = [&](int i) { return corner(p, face(i), at(i) + 1); };
  auto prv = [&](int i) { return corner(p, face(i), at(i) + 2); };
  bool frozen = false;
  int starts = 0, first = -1;
  for (int i = 0; i < k && !frozen; i++) {
    int cn = 0, cp = 0;
    bool ends = false;
    for (int m = 0; m < k; m++) {
      cn += nxt(m) == nxt(i);
      cp += prv(m) == prv(i);
      ends = ends || prv(m) == nxt(i);
    }
    frozen = cn > 1 || cp > 1;
    if (!ends && starts++ == 0) first = i;
  }
  if (!frozen && starts > 1) frozen = true;
  if (!frozen) {
    if (first < 0) first = 0;
    int i = first, count = 1;
    while (count <= k) {
      int j = -1;
      for (int m = 0; m < k && j < 0; m++)
        if (nxt(m) == prv(i)) j = m;
      if (j < 0 || j == first) break;
      i = j;
      count++;
    }
    frozen = count < k;
  }
  if (frozen) {
    p.frozen[x] = 1;
    atomicAdd(&p.res->frozen, 1u);
    return;
  }
  double area = 0.0;
  for (int pass = 0; pass < 2; pass++)
    for (int i = 0; i < k; i++) {
      const int t = face(i);
      const D3 p0 = vertex_of(p.pos, corner(p, t, 0)), p1 = vertex_of(p.pos, corner(p, t, 1)),
               p2 = vertex_of(p.pos, corner(p, t, 2));
      const D3 n = normal3(p0, p1, p2);
      const double ln = sqrt(dot3(n, n));
      if (!(ln > 0.0)) continue;
      const D3 un = {n.x / ln, n.y / ln, n.z / ln};
      if (pass == 0) {
        const double fa = 0.5 * ln;
        plane_add(q, un, -dot3(un, p0), fa);
        area = area + fa;
        continue;
      }
      for (int e = 0; e < 3; e++) {
        const int a = corner(p, t, e), b = corner(p, t, e + 1);
        if ((a != x && b != x) || has_directed(p, x, b, a)) continue;
        const D3 pa = vertex_of(p.pos, a), ev = sub3(vertex_of(p.pos, b), pa);
        const D3 m = cross3(ev, un);
        const double lm = sqrt(dot3(m, m));
        if (!(lm > 0.0)) continue;
        const D3 mu = {m.x / lm, m.y / lm, m.z / lm};
        plane_add(q, mu, -dot3(mu, pa), p.bw * dot3(ev, ev));
      }
    }
  p.A[x] = area;
}

// ---- a pass -----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MT) simplify_candidate_kernel(SimplifyParams p)
{
  unsigned int n = 0;
  for (int c = blockIdx.x * MT + threadIdx.x; c < 3 * p.T; c += gridDim.x * MT) {
    const int t = c / 3, k = c - 3 * t;
    int u, v, drops = 0;
    D3 x;
    double err;
    unsigned long long key = NO_KEY;
    if (evaluate(p, t, k, u, v, x, err, drops)) {
      key = ((unsigned long long)__float_as_uint(__double2float_rn(err)) << 32) |
            tie_of((unsigned int)(3 * p.tid[t] + k));
      n++;
    }
    p.key[c] = key;
    p.drops[c] = drops;
  }
  if (n) atomicAdd(&p.res->cand, n);
}

__global__ void simplify_threshold_kernel(SimplifyParams p)
{
  const unsigned int C = p.res->cand;
  const unsigned int m = (C + (1u << F_SHIFT) - 1) >> F_SHIFT;
  p.res->thr = C ? p.keyS[m - 1] : 0ull;
}

template <class F>
__device__ __forceinline__ void closed_rings(const SimplifyParams &p, int c, F &&f)
{
  const int t = c / 3, k = c - 3 * t;
  const int ends[2] = {corner(p, t, k), corner(p, t, k + 1)};
  for (int e = 0; e < 2; e++)
    any_face(p, ends[e], [&](int s, int) {
      for (int j = 0; j < 3; j++) f(corner(p, s, j));
      return false;
    });
}

__global__ void __launch_bounds__(MT) simplify_scatter_kernel(SimplifyParams p)
{
  const unsigned long long thr = p.res->thr;
  for (int c = blockIdx.x * MT + threadIdx.x; c < 3 * p.T; c += gridDim.x * MT) {
    const unsigned long long key = p.key[c];
    if (key == NO_KEY || key > thr) continue;
    closed_rings(p, c, [&](int w) { atomicMin(&p.mark[w], key); });
  }
}

__global__ void __launch_bounds__(MT) simplify_select_kernel(SimplifyParams p)
{
  const unsigned long long thr = p.res->thr;
  unsigned int ns = 0, nd = 0;
  for (int c = blockIdx.x * MT + threadIdx.x; c < 3 * p.T; c += gridDim.x * MT) {
    const unsigned long long key = p.key[c];
    bool sel = key != NO_KEY && key <= thr;
    if (sel) closed_rings(p, c, [&](int w) { sel = sel && p.mark[w] == key; });
    p.selKey[c] = sel ? key : NO_KEY;
    if (!sel) p.drops[c] = 0;
    ns += sel;
    nd += sel ? p.drops[c] : 0;
  }
  if (ns) {
    atomicAdd(&p.res->sel, ns);
    atomicAdd(&p.res->drops, nd);
  }
}

// the target pass: the selected edges by key, their faces summed; the last applied is where the sum reaches need
__global__ void __launch_bounds__(MT) simplify_cut_kernel(SimplifyParams p, int need)
{
  const int S = (int)p.res->sel;
  for (int i = blockIdx.x * MT + threadIdx.x; i < S; i += gridDim.x * MT)
    if (p.cum[i] >= need && (i == 0 || p.cum[i - 1] < need)) {
      p.res->cut = p.selKeyS[i];
      p.res->applied = i + 1;
    }
}

__global__ void __launch_bounds__(MT) simplify_collapse_kernel(SimplifyParams p)
{
  const unsigned long long cut = p.res->cut;
  for (int c = blockIdx.x * MT + threadIdx.x; c < 3 * p.T; c += gridDim.x * MT) {
    const unsigned long long key = p.selKey[c];
    if (key == NO_KEY || key > cut) continue;
    const int t = c / 3, k = c - 3 * t;
    int u, v, drops;
    D3 x;
    double err;
    if (!evaluate(p, t, k, u, v, x, err, drops)) continue;   // cannot happen: the state it read is unchanged
    const D3 pu = vertex_of(p.pos, u), pv = vertex_of(p.pos, v);
    if (p.inten) {
      const D3 d = sub3(pv, pu);
      const double den = dot3(d, d);
      double s = den > 0.0 ? dot3(sub3(x, pu), d) / den : 0.0;
      s = !(s > 0.0) ? 0.0 : (s > 1.0 ? 1.0 : s);
      const double iu = p.inten[u], iv = p.inten[v];
      p.inten[u] = __double2float_rn(iu + s * (iv - iu));
    }
    p.pos[3 * (size_t)u] = x.x;
    p.pos[3 * (size_t)u + 1] = x.y;
    p.pos[3 * (size_t)u + 2] = x.z;
    for (int i = 0; i < 10; i++) p.Q[10 * (size_t)u + i] = p.Q[10 * (size_t)u + i] + p.Q[10 * (size_t)v + i];
    p.A[u] = p.A[u] + p.A[v];
    p.remap[v] = u;
    atomicMax(&p.res->maxErr, (unsigned long long)__double_as_longlong(err));
  }
}

__device__ __forceinline__ bool kept_face(const SimplifyParams &p, int t, int *g)
{
  for (int j = 0; j < 3; j++) g[j] = p.remap[p.tri[3 * (size_t)t + j]];
  return g[0] != g[1] && g[1] != g[2] && g[0] != g[2];
}

__global__ void __launch_bounds__(MT) simplify_face_count_kernel(SimplifyParams p)
{
  const int t = blockIdx.x * MT + threadIdx.x;
  int g[3];
  counted_cta_count<MT>(t < p.T && kept_face(p, t, g) ? 1 : 0, p.blockCounts + blockIdx.x);
}

__global__ void __launch_bounds__(MT) simplify_face_write_kernel(SimplifyParams p)
{
  const int t = blockIdx.x * MT + threadIdx.x;
  int g[3];
  const bool keep = t < p.T && kept_face(p, t, g);
  const int at = p.blockOffsets[blockIdx.x] + counted_position<MT>(keep ? 1 : 0);
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0)
    p.res->tris = counted_total(p.blockOffsets, p.blockCounts, gridDim.x - 1);
  if (!keep) return;
  for (int j = 0; j < 3; j++) p.triN[3 * (size_t)at + j] = g[j];
  p.tidN[at] = p.tid[t];
}

// ---- output -----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MT) simplify_used_kernel(SimplifyParams p)
{
  for (int c = blockIdx.x * MT + threadIdx.x; c < 3 * p.T; c += gridDim.x * MT) p.used[p.tri[c]] = 1;
}

__global__ void __launch_bounds__(MT) simplify_vcount_kernel(SimplifyParams p)
{
  const int x = blockIdx.x * MT + threadIdx.x;
  counted_cta_count<MT>(x < p.V ? p.used[x] : 0, p.blockCounts + blockIdx.x);
}

// the used vertices in ascending input index; used[] becomes the output index
__global__ void __launch_bounds__(MT) simplify_vwrite_kernel(SimplifyParams p)
{
  const int x = blockIdx.x * MT + threadIdx.x;
  const int u = x < p.V ? p.used[x] : 0;
  const int at = p.blockOffsets[blockIdx.x] + counted_position<MT>(u);
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0)
    p.res->verts = counted_total(p.blockOffsets, p.blockCounts, gridDim.x - 1);
  if (!u) return;
  p.used[x] = at;
  if (at >= p.maxOutV) return;
  for (int d = 0; d < 3; d++) p.outV[3 * (size_t)at + d] = __double2float_rn(p.pos[3 * (size_t)x + d]);
  if (p.outI) p.outI[at] = p.inten[x];
}

__global__ void __launch_bounds__(MT) simplify_twrite_kernel(SimplifyParams p)
{
  const int t = blockIdx.x * MT + threadIdx.x;
  if (t >= p.T || t >= p.maxOutT) return;
  for (int j = 0; j < 3; j++) p.outT[3 * (size_t)t + j] = p.used[p.tri[3 * (size_t)t + j]];
}

}  // namespace

int simplify_run(const float *vin, const float *iin, int V, const int *tin, int T0, int target, double maxError,
                 double bw, float *outV, float *outI, int maxOutV, int *outT, int maxOutT, cudaStream_t st,
                 void *h_res, double *info, long long *stats)
{
  const size_t C3 = 3 * (size_t)T0;
  const int nbT = idivup(std::max(T0, 1), MT), nbV = idivup(std::max(V, 1), MT);
  const int vbits = radix_bits(std::max(V, 1));
  size_t tb[7] = {};
  CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb[0], (int *)nullptr, (int *)nullptr, (int *)nullptr,
                                          (int *)nullptr, (int)C3, 0, vbits, st));
  CS_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb[1], (unsigned long long *)nullptr,
                                         (unsigned long long *)nullptr, (int)C3, 0, 64, st));
  CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb[2], (unsigned long long *)nullptr,
                                          (unsigned long long *)nullptr, (int *)nullptr, (int *)nullptr, (int)C3, 0,
                                          64, st));
  CS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb[3], (int *)nullptr, (int *)nullptr, V + 1, st));
  CS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb[4], (int *)nullptr, (int *)nullptr, std::max(nbT, nbV), st));
  CS_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tb[5], (int *)nullptr, (int *)nullptr, (int)C3, st));
  size_t tempBytes = 0;
  for (size_t b : tb) tempBytes = std::max(tempBytes, b);

  Layout L(256);
  const size_t resAt = L.take(sizeof(SimplifyResult));
  const size_t triAt = L.take(C3 * 4), triNAt = L.take(C3 * 4), tidAt = L.take((size_t)T0 * 4),
               tidNAt = L.take((size_t)T0 * 4);
  const size_t ckAt = L.take(C3 * 4), ckSAt = L.take(C3 * 4), cvAt = L.take(C3 * 4), cvSAt = L.take(C3 * 4);
  const size_t keyAt = L.take(C3 * 8), keySAt = L.take(C3 * 8), selAt = L.take(C3 * 8), selSAt = L.take(C3 * 8);
  const size_t drAt = L.take(C3 * 4), drSAt = L.take(C3 * 4), cumAt = L.take(C3 * 4);
  const size_t cntAt = L.take(((size_t)V + 1) * 4), startAt = L.take(((size_t)V + 1) * 4);
  const size_t posAt = L.take((size_t)V * 24), qAt = L.take((size_t)V * 80), aAt = L.take((size_t)V * 8);
  const size_t inAt = iin ? L.take((size_t)V * 4) : 0;
  const size_t frAt = L.take((size_t)V), remapAt = L.take((size_t)V * 4), usedAt = L.take((size_t)V * 4);
  const size_t markAt = L.take((size_t)V * 8);
  const size_t bcAt = L.take((size_t)std::max(nbT, nbV) * 4), boAt = L.take((size_t)std::max(nbT, nbV) * 4);
  const size_t tempAt = L.take(tempBytes);
  char *base = nullptr;
  CS_CUDA(cudaMallocAsync((void **)&base, L.bytes, st));
  auto at = [&](size_t off) { return base + off; };

  SimplifyParams p{};
  p.res = reinterpret_cast<SimplifyResult *>(at(resAt));
  p.V = V;
  p.T = T0;
  p.vin = vin;
  p.iin = iin;
  p.tin = tin;
  p.tri = reinterpret_cast<int *>(at(triAt));
  p.triN = reinterpret_cast<int *>(at(triNAt));
  p.tid = reinterpret_cast<int *>(at(tidAt));
  p.tidN = reinterpret_cast<int *>(at(tidNAt));
  p.ckey = reinterpret_cast<int *>(at(ckAt));
  p.ckeyS = reinterpret_cast<int *>(at(ckSAt));
  p.cval = reinterpret_cast<int *>(at(cvAt));
  p.cvalS = reinterpret_cast<int *>(at(cvSAt));
  p.vcount = reinterpret_cast<int *>(at(cntAt));
  p.vstart = reinterpret_cast<int *>(at(startAt));
  p.pos = reinterpret_cast<double *>(at(posAt));
  p.Q = reinterpret_cast<double *>(at(qAt));
  p.A = reinterpret_cast<double *>(at(aAt));
  p.inten = iin ? reinterpret_cast<float *>(at(inAt)) : nullptr;
  p.frozen = reinterpret_cast<unsigned char *>(at(frAt));
  p.remap = reinterpret_cast<int *>(at(remapAt));
  p.used = reinterpret_cast<int *>(at(usedAt));
  p.key = reinterpret_cast<unsigned long long *>(at(keyAt));
  p.keyS = reinterpret_cast<unsigned long long *>(at(keySAt));
  p.selKey = reinterpret_cast<unsigned long long *>(at(selAt));
  p.selKeyS = reinterpret_cast<unsigned long long *>(at(selSAt));
  p.mark = reinterpret_cast<unsigned long long *>(at(markAt));
  p.drops = reinterpret_cast<int *>(at(drAt));
  p.dropsS = reinterpret_cast<int *>(at(drSAt));
  p.cum = reinterpret_cast<int *>(at(cumAt));
  p.blockCounts = reinterpret_cast<int *>(at(bcAt));
  p.blockOffsets = reinterpret_cast<int *>(at(boAt));
  p.bw = bw;
  p.maxError = maxError;
  p.outV = outV;
  p.outI = outI;
  p.outT = outT;
  p.maxOutV = maxOutV;
  p.maxOutT = maxOutT;
  void *temp = at(tempAt);
  SimplifyResult &R = *static_cast<SimplifyResult *>(h_res);
  cudaEvent_t *tev = match_timing_events();

  int status = 0, passes = 0;
  long long collapses = 0;
  auto readback = [&]() -> int {
    CS_CUDA(cudaMemcpyAsync(h_res, p.res, sizeof(SimplifyResult), cudaMemcpyDeviceToHost, st));
    CS_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  auto adjacency = [&]() -> int {
    CS_CUDA(cudaMemsetAsync(p.vcount, 0, ((size_t)V + 1) * 4, st));
    simplify_corners_kernel<<<grid_of(3ll * p.T), MT, 0, st>>>(p);
    count_launch();
    CS_CUDA(cudaGetLastError());
    CS_CUDA(cub::DeviceRadixSort::SortPairs(temp, tempBytes, p.ckey, p.ckeyS, p.cval, p.cvalS, 3 * p.T, 0, vbits, st));
    CS_CUDA(cub::DeviceScan::ExclusiveSum(temp, tempBytes, p.vcount, p.vstart, V + 1, st));
    return 0;
  };
  auto run = [&]() -> int {
    int r;
    if (tev) CS_CUDA(cudaEventRecord(tev[0], st));
    CS_CUDA(cudaMemsetAsync(p.res, 0, sizeof(SimplifyResult), st));
    mesh_validate_kernel<<<grid_of(T0), MT, 0, st>>>(vin, V, tin, T0, &p.res->bad);
    count_launch();
    CS_CUDA(cudaGetLastError());
    if ((r = readback()) < 0) return r;
    if (R.bad) {
      status = 2;
      return 0;
    }
    simplify_init_kernel<<<grid_of(std::max(V, T0)), MT, 0, st>>>(p);
    count_launch();
    CS_CUDA(cudaGetLastError());
    if ((r = adjacency()) < 0) return r;
    simplify_vertex_kernel<<<nbV, MT, 0, st>>>(p);
    count_launch();
    CS_CUDA(cudaGetLastError());
    if (tev) CS_CUDA(cudaEventRecord(tev[1], st));
    for (;;) {
      if (p.T <= target) { status = 0; break; }
      if (passes == MAX_PASSES) { status = 3; break; }
      const long long C = 3ll * p.T;
      CS_CUDA(cudaMemsetAsync(&p.res->cand, 0, 3 * sizeof(unsigned int), st));
      CS_CUDA(cudaMemsetAsync(&p.res->cut, 0xff, sizeof(unsigned long long), st));
      CS_CUDA(cudaMemsetAsync(p.mark, 0xff, (size_t)V * 8, st));
      simplify_candidate_kernel<<<grid_of(C), MT, 0, st>>>(p);
      CS_CUDA(cub::DeviceRadixSort::SortKeys(temp, tempBytes, p.key, p.keyS, (int)C, 0, 64, st));
      simplify_threshold_kernel<<<1, 1, 0, st>>>(p);
      simplify_scatter_kernel<<<grid_of(C), MT, 0, st>>>(p);
      simplify_select_kernel<<<grid_of(C), MT, 0, st>>>(p);
      count_launch(4);
      CS_CUDA(cudaGetLastError());
      if ((r = readback()) < 0) return r;
      if (R.cand == 0) { status = 1; break; }
      bool last = false;
      if ((long long)p.T - R.drops < target) {
        const int need = p.T - target;
        CS_CUDA(cub::DeviceRadixSort::SortPairs(temp, tempBytes, p.selKey, p.selKeyS, p.drops, p.dropsS, (int)C, 0,
                                                64, st));
        CS_CUDA(cub::DeviceScan::InclusiveSum(temp, tempBytes, p.dropsS, p.cum, (int)R.sel, st));
        simplify_cut_kernel<<<grid_of(R.sel), MT, 0, st>>>(p, need);
        count_launch();
        CS_CUDA(cudaGetLastError());
        last = true;
      }
      simplify_collapse_kernel<<<grid_of(C), MT, 0, st>>>(p);
      const int nb = idivup(p.T, MT);
      simplify_face_count_kernel<<<nb, MT, 0, st>>>(p);
      count_launch(2);
      CS_CUDA(cudaGetLastError());
      CS_CUDA(cub::DeviceScan::ExclusiveSum(temp, tempBytes, p.blockCounts, p.blockOffsets, nb, st));
      simplify_face_write_kernel<<<nb, MT, 0, st>>>(p);
      count_launch();
      CS_CUDA(cudaGetLastError());
      std::swap(p.tri, p.triN);
      std::swap(p.tid, p.tidN);
      passes++;
      if (last) {
        if ((r = readback()) < 0) return r;
        collapses += R.applied;
        p.T = (int)R.tris;
      } else {
        collapses += R.sel;
        p.T -= (int)R.drops;
      }
      if ((r = adjacency()) < 0) return r;
    }
    if (tev) CS_CUDA(cudaEventRecord(tev[2], st));
    CS_CUDA(cudaMemsetAsync(p.used, 0, (size_t)V * 4, st));
    simplify_used_kernel<<<grid_of(3ll * p.T), MT, 0, st>>>(p);
    simplify_vcount_kernel<<<nbV, MT, 0, st>>>(p);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    CS_CUDA(cub::DeviceScan::ExclusiveSum(temp, tempBytes, p.blockCounts, p.blockOffsets, nbV, st));
    simplify_vwrite_kernel<<<nbV, MT, 0, st>>>(p);
    simplify_twrite_kernel<<<idivup(std::max(p.T, 1), MT), MT, 0, st>>>(p);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    if ((r = readback()) < 0) return r;
    if (tev) {
      CS_CUDA(cudaEventRecord(tev[3], st));
      static const char *const names[3] = {"setup", "passes", "output"};
      report_stage_times(tev, names, 3, "simplify timing triangles=%d passes=%d", T0, passes);
    }
    return 0;
  };
  const int r = run();
  cudaFreeAsync(base, st);
  if (r < 0) return r;
  const bool out = status != 2;
  const long long Vout = out ? R.verts : 0, Tout = out ? p.T : 0;
  double maxErr = 0.0;
  std::memcpy(&maxErr, &R.maxErr, sizeof maxErr);
  if (info) info[0] = out ? std::sqrt(maxErr) : 0.0;
  if (stats) {
    stats[0] = T0;
    stats[1] = out ? R.frozen : 0;
    stats[2] = passes;
    stats[3] = collapses;
    stats[4] = Vout;
    stats[5] = Tout;
    stats[6] = std::min(Vout, (long long)maxOutV);
    stats[7] = std::min(Tout, (long long)maxOutT);
    stats[8] = status;
  }
  return (int)Tout;
}

size_t simplify_result_bytes() { return sizeof(SimplifyResult); }

}  // namespace cs
