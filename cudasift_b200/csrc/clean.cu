// clean.cu -- mesh cleaning (cs_clean_mesh) in count-scan-write passes: degenerate faces and duplicate vertex sets by a
// two-key radix sort of each face's sorted ids, one radix sort of the undirected edge keys whose runs serve the
// long-edge statistics (coop.cuh's three-level totals), the non-manifold edges, the component links (common.cuh's
// union-find) and the boundary half-edges; the boundary loops by pointer jumping over the listed half-edges, ear
// cutting one thread per loop, Taubin smoothing over sorted directed edge keys, and the output lists of
// counted_list.cuh.  Every rule is stated in cudasift_b200.h at cs_clean_mesh; tests/clean_oracle.py restates them in
// float64.
//
// Determinism: no floating-point atomics; integer atomics only where the result does not depend on their order
// (counts, component sizes, the largest size, the union-find hooks of common.cuh).  A face dropped by rule 4 is marked
// in a separate array and dropped after the pass, so no run reads another run's writes.  This unit is compiled with
// -fmad=false so that every float64 product and sum is rounded once, in the order written, as the oracle computes it.
#include <cmath>
#include <cstring>

#include <cub/cub.cuh>

#include "common.cuh"
#include "coop.cuh"
#include "counted_list.cuh"
#include "trimesh.cuh"

namespace cs {

namespace {

constexpr int MAX_HOLE = 256;                 // the longest loop that is filled

// The device words of a call.
struct CleanResult {
  unsigned int bad;                           // an invalid input (status 2)
  unsigned int degenerate, duplicate, longEdge, nonManifold, small;   // faces dropped by rules 2 to 5
  unsigned int components, removed, largest, nmVertices;              // rule 5 and the non-manifold vertices
  unsigned int loops, filled, chain;          // rule 6: cycles, filled cycles, half-edges on no cycle
  int bnd;                                    // boundary half-edges listed
  int kept, fill, tris, verts;                // kept input faces, fill faces, all faces, output vertices
  double mean, sdev, thr;                     // rule 3
};

struct CleanParams {
  CleanResult *res;
  int V, T;
  const float *vin, *iin;                     // input vertices [V][3], intensities [V] (or null)
  const int *tin;                             // input triangles [T][3]
  int *alive, *drop;                          // [T] face kept so far, rule 4's marks
  int *parent, *size;                         // [T] face union-find, component sizes at the roots
  int *cparent;                               // [3T] corner union-find (the fans of a vertex)
  int *fans;                                  // [V] fans per vertex
  int *k1, *fv, *fvS, *fv2S;                  // [T] rule 2: the highest sorted id and the faces
  unsigned long long *k2;                     // [T] rule 2: (lowest << 32) | middle sorted id
  unsigned long long *ekey, *ekeyS;           // [3T] undirected edge keys of every input face, and sorted (ekey
                                              // is then the key output of rule 2's sorts)
  int *ec, *ecS;                              // [3T] their corners
  double *part, *group;                       // three-level total partials
  int *bflag, *blist, *nxt, *J, *Jn, *M, *Mn; // [3T] boundary half-edges, successors and jumps
  int *hin, *hout, *outH;                     // [V] boundary half-edges in and out of a vertex, the out half-edge
  int *fcnt, *foff, *hstart, *okc, *fpos;     // [V + 1] per loop start vertex: fill faces, offsets, start, kept
  int *fillS;                                 // [3T][3] fill faces of every loop
  int *ftri;                                  // [4T][3] the output faces (kept input faces, then fill faces)
  unsigned long long *dkey, *dkeyS;           // [6 tris] directed edge keys and sorted (smoothing)
  int *vfirst, *vend;                         // [V] a vertex's range of sorted directed keys
  unsigned char *fixed;                       // [V]
  double *pos, *posN;                         // [V][3]
  int *used;                                  // [V]
  int *blockCounts, *blockOffsets;
  int minFaces, maxHole;
  double minFraction, longFactor;
  float *outV, *outI;
  int *outT;
  int maxOutV, maxOutT;
};

__device__ __forceinline__ int nextc(int c) { const int t = c / 3; return 3 * t + (c - 3 * t + 1) % 3; }
__device__ __forceinline__ D3 P(const CleanParams &p, int v) { return vertex_of(p.vin, v); }
__device__ __forceinline__ double edge_len(const CleanParams &p, int a, int b)
{
  const D3 d = sub3(P(p, b), P(p, a));
  return sqrt(dot3(d, d));
}
// the boundary half-edge h of the list runs from the next corner's vertex to its corner's vertex
__device__ __forceinline__ int h_from(const CleanParams &p, int h) { return p.tin[nextc(p.blist[h])]; }
__device__ __forceinline__ int h_to(const CleanParams &p, int h) { return p.tin[p.blist[h]]; }
__device__ __forceinline__ bool run_head(const unsigned long long *k, int i) { return i == 0 || k[i - 1] != k[i]; }
// the first sorted position of the edge {a, b} (a binary search; 3T when no input face holds it)
__device__ __forceinline__ int edge_lower(const CleanParams &p, int a, int b)
{
  const unsigned long long k = ((unsigned long long)min(a, b) << 32) | (unsigned int)max(a, b);
  int lo = 0, hi = 3 * p.T;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (p.ekeyS[mid] < k) lo = mid + 1; else hi = mid;
  }
  return lo < 3 * p.T && p.ekeyS[lo] == k ? lo : 3 * p.T;
}
// f(face, corner) for every face of the edge run at sorted position i that is still alive, in ascending face index;
// returns their count
template <class F>
__device__ __forceinline__ int run_alive(const CleanParams &p, int i, F &&f)
{
  const unsigned long long k = p.ekeyS[i];
  int n = 0;
  for (int j = i; j < 3 * p.T && p.ekeyS[j] == k; j++) {
    const int c = p.ecS[j], t = c / 3;
    if (p.alive[t]) f(t, c, n++);
  }
  return n;
}

// ---- setup and rule 2 -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MT) clean_init_kernel(CleanParams p)
{
  const int n = max(p.V, 3 * p.T);
  for (int i = blockIdx.x * MT + threadIdx.x; i < n; i += gridDim.x * MT) {
    if (i < p.V)
      for (int d = 0; d < 3; d++) p.pos[3 * (size_t)i + d] = (double)p.vin[3 * (size_t)i + d];
    if (i < p.T) {
      p.alive[i] = 1;
      p.parent[i] = i;
    }
    if (i < 3 * p.T) p.cparent[i] = i;
  }
}

__device__ __forceinline__ void sorted_ids(const int *tin, int t, unsigned int &s0, unsigned int &s1, unsigned int &s2)
{
  const unsigned int a = tin[3 * (size_t)t], b = tin[3 * (size_t)t + 1], c = tin[3 * (size_t)t + 2];
  s0 = min(a, min(b, c));
  s2 = max(a, max(b, c));
  s1 = a ^ b ^ c ^ s0 ^ s2;
}

// every edge of face t is held by another input face
__device__ bool enclosed(const CleanParams &p, int t)
{
  for (int k = 0; k < 3; k++) {
    const int i = edge_lower(p, p.tin[3 * t + k], p.tin[3 * t + (k + 1) % 3]);
    if (i + 1 >= 3 * p.T || p.ekeyS[i + 1] != p.ekeyS[i]) return false;
  }
  return true;
}

// rule 2a: n.n == 0 drops the face unless it is enclosed; the first sort key is the highest sorted id
__global__ void __launch_bounds__(MT) clean_face_key_kernel(CleanParams p)
{
  unsigned int n = 0;
  for (int t = blockIdx.x * MT + threadIdx.x; t < p.T; t += gridDim.x * MT) {
    const D3 nr = normal3(P(p, p.tin[3 * t]), P(p, p.tin[3 * t + 1]), P(p, p.tin[3 * t + 2]));
    if (dot3(nr, nr) == 0.0 && !enclosed(p, t)) {
      p.alive[t] = 0;
      n++;
    }
    unsigned int s0, s1, s2;
    sorted_ids(p.tin, t, s0, s1, s2);
    p.k1[t] = (int)s2;
    p.fv[t] = t;
  }
  if (n) atomicAdd(&p.res->degenerate, n);
}

// the second key, (lowest << 32) | middle, in the order of the first sort
__global__ void __launch_bounds__(MT) clean_face_key2_kernel(CleanParams p)
{
  for (int i = blockIdx.x * MT + threadIdx.x; i < p.T; i += gridDim.x * MT) {
    unsigned int s0, s1, s2;
    sorted_ids(p.tin, p.fvS[i], s0, s1, s2);
    p.k2[i] = ((unsigned long long)s0 << 32) | s1;
  }
}

// rule 2b: in a run of equal vertex sets (faces ascending), the first face still alive stays, the others go
__global__ void __launch_bounds__(MT) clean_duplicate_kernel(CleanParams p)
{
  unsigned int n = 0;
  for (int i = blockIdx.x * MT + threadIdx.x; i < p.T; i += gridDim.x * MT) {
    unsigned int a0, a1, a2, b0, b1, b2;
    sorted_ids(p.tin, p.fv2S[i], a0, a1, a2);
    if (i > 0) {
      sorted_ids(p.tin, p.fv2S[i - 1], b0, b1, b2);
      if (a0 == b0 && a1 == b1 && a2 == b2) continue;
    }
    bool first = true;
    for (int j = i; j < p.T; j++) {
      const int t = p.fv2S[j];
      sorted_ids(p.tin, t, b0, b1, b2);
      if (a0 != b0 || a1 != b1 || a2 != b2) break;
      if (!p.alive[t]) continue;
      if (first) {
        first = false;
      } else {
        p.alive[t] = 0;
        n++;
      }
    }
  }
  if (n) atomicAdd(&p.res->duplicate, n);
}

__global__ void __launch_bounds__(MT) clean_edge_key_kernel(CleanParams p)
{
  for (int c = blockIdx.x * MT + threadIdx.x; c < 3 * p.T; c += gridDim.x * MT) {
    p.ekey[c] = edge_key_of(p.tin, c);
    p.ec[c] = c;
  }
}

// ---- rule 3 -----------------------------------------------------------------------------------------------------------
// (1, l, l^2) of every distinct edge of the kept faces, at its run head, in coop.cuh's three-level order
__global__ void __launch_bounds__(MT) clean_edge_tiles_kernel(CleanParams p)
{
  co_tree_tiles<3, MT>(3 * p.T, p.part, [&](int i, double *v) {
    if (!run_head(p.ekeyS, i) || run_alive(p, i, [](int, int, int) {}) == 0) return;
    const unsigned long long k = p.ekeyS[i];
    const double l = edge_len(p, (int)(k >> 32), (int)(k & 0xffffffffu));
    v[0] = v[0] + 1.0;
    v[1] = v[1] + l;
    v[2] = v[2] + l * l;
  });
}

__global__ void __launch_bounds__(MT) clean_edge_groups_kernel(CleanParams p)
{
  co_tree_groups<3, MT>(3 * p.T, p.part, p.group);
}

__global__ void __launch_bounds__(MT) clean_edge_total_kernel(CleanParams p)
{
  double tot[3];
  co_tree_total<3, MT>(3 * p.T, p.group, tot);
  if (threadIdx.x != 0) return;
  double m = 0.0, s = 0.0;
  if (tot[0] > 0.0) {
    m = tot[1] / tot[0];
    const double var = tot[2] / tot[0] - m * m;
    s = var > 0.0 ? sqrt(var) : 0.0;
  }
  p.res->mean = m;
  p.res->sdev = s;
  p.res->thr = m + p.longFactor * s;
}

__global__ void __launch_bounds__(MT) clean_long_kernel(CleanParams p)
{
  const double thr = p.res->thr;
  unsigned int n = 0;
  for (int t = blockIdx.x * MT + threadIdx.x; t < p.T; t += gridDim.x * MT) {
    if (!p.alive[t]) continue;
    const int a = p.tin[3 * t], b = p.tin[3 * t + 1], c = p.tin[3 * t + 2];
    if (edge_len(p, min(a, b), max(a, b)) > thr || edge_len(p, min(b, c), max(b, c)) > thr ||
        edge_len(p, min(c, a), max(c, a)) > thr) {
      p.alive[t] = 0;
      n++;
    }
  }
  if (n) atomicAdd(&p.res->longEdge, n);
}

// ---- rule 4 -----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MT) clean_fin_mark_kernel(CleanParams p)
{
  for (int i = blockIdx.x * MT + threadIdx.x; i < 3 * p.T; i += gridDim.x * MT)
    if (run_head(p.ekeyS, i))
      run_alive(p, i, [&](int t, int, int k) {
        if (k >= 2) p.drop[t] = 1;
      });
}

__global__ void __launch_bounds__(MT) clean_fin_drop_kernel(CleanParams p)
{
  unsigned int n = 0;
  for (int t = blockIdx.x * MT + threadIdx.x; t < p.T; t += gridDim.x * MT)
    if (p.drop[t] && p.alive[t]) {
      p.alive[t] = 0;
      n++;
    }
  if (n) atomicAdd(&p.res->nonManifold, n);
}

// ---- rule 5 and the non-manifold vertices -----------------------------------------------------------------------------
// an edge of exactly two faces joins the faces, and the corners of each of its ends
__global__ void __launch_bounds__(MT) clean_link_kernel(CleanParams p)
{
  for (int i = blockIdx.x * MT + threadIdx.x; i < 3 * p.T; i += gridDim.x * MT) {
    if (!run_head(p.ekeyS, i)) continue;
    int cs[2] = {-1, -1};
    const int n = run_alive(p, i, [&](int, int c, int k) {
      if (k < 2) cs[k] = c;
    });
    if (n != 2) continue;
    const int c1 = cs[0], c2 = cs[1], n1 = nextc(c1), n2 = nextc(c2);
    uf_link(p.parent, c1 / 3, c2 / 3);
    if (p.tin[c1] == p.tin[c2]) {
      uf_link(p.cparent, c1, c2);
      uf_link(p.cparent, n1, n2);
    } else {
      uf_link(p.cparent, c1, n2);
      uf_link(p.cparent, n1, c2);
    }
  }
}

__global__ void __launch_bounds__(MT) clean_roots_kernel(CleanParams p)
{
  for (int t = blockIdx.x * MT + threadIdx.x; t < p.T; t += gridDim.x * MT) {
    if (!p.alive[t]) continue;
    atomicAdd(&p.size[uf_find(p.parent, t)], 1);
    for (int k = 0; k < 3; k++)
      if (uf_find(p.cparent, 3 * t + k) == 3 * t + k) atomicAdd(&p.fans[p.tin[3 * t + k]], 1);
  }
}

__global__ void __launch_bounds__(MT) clean_count_kernel(CleanParams p)
{
  unsigned int nc = 0, nv = 0;
  for (int i = blockIdx.x * MT + threadIdx.x; i < max(p.T, p.V); i += gridDim.x * MT) {
    if (i < p.T && p.alive[i] && p.parent[i] == i) {
      nc++;
      atomicMax(&p.res->largest, (unsigned int)p.size[i]);
    }
    if (i < p.V && p.fans[i] > 1) nv++;
  }
  if (nc) atomicAdd(&p.res->components, nc);
  if (nv) atomicAdd(&p.res->nmVertices, nv);
}

__global__ void __launch_bounds__(MT) clean_small_kernel(CleanParams p)
{
  const double largest = (double)p.res->largest;
  unsigned int nf = 0, nr = 0;
  for (int t = blockIdx.x * MT + threadIdx.x; t < p.T; t += gridDim.x * MT) {
    if (!p.alive[t]) continue;
    const int r = uf_find(p.parent, t), s = p.size[r];
    if (s < p.minFaces || (double)s < p.minFraction * largest) {
      p.alive[t] = 0;
      nf++;
      nr += r == t;
    }
  }
  if (nf) atomicAdd(&p.res->small, nf);
  if (nr) atomicAdd(&p.res->removed, nr);
}

// ---- rule 6: boundary loops ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MT) clean_boundary_kernel(CleanParams p)
{
  for (int i = blockIdx.x * MT + threadIdx.x; i < 3 * p.T; i += gridDim.x * MT) {
    if (!run_head(p.ekeyS, i)) continue;
    int c = -1;
    if (run_alive(p, i, [&](int, int cc, int) { c = cc; }) != 1) continue;
    p.bflag[c] = 1;
    atomicAdd(&p.hout[p.tin[nextc(c)]], 1);
    atomicAdd(&p.hin[p.tin[c]], 1);
  }
}

__global__ void __launch_bounds__(MT) clean_bcount_kernel(CleanParams p)
{
  const int c = blockIdx.x * MT + threadIdx.x;
  counted_cta_count<MT>(c < 3 * p.T ? p.bflag[c] : 0, p.blockCounts + blockIdx.x);
}

// the boundary half-edges in ascending corner order; a vertex with one outgoing half-edge records it
__global__ void __launch_bounds__(MT) clean_bwrite_kernel(CleanParams p)
{
  const int c = blockIdx.x * MT + threadIdx.x;
  const int f = c < 3 * p.T ? p.bflag[c] : 0;
  const int at = p.blockOffsets[blockIdx.x] + counted_position<MT>(f);
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0)
    p.res->bnd = (int)counted_total(p.blockOffsets, p.blockCounts, gridDim.x - 1);
  if (!f) return;
  p.blist[at] = c;
  const int from = p.tin[nextc(c)];
  if (p.hout[from] == 1) p.outH[from] = at;
}

// successor: the out half-edge at the end vertex when that vertex has one boundary half-edge in and one out
__global__ void __launch_bounds__(MT) clean_succ_kernel(CleanParams p)
{
  const int B = p.res->bnd;
  for (int h = blockIdx.x * MT + threadIdx.x; h < B; h += gridDim.x * MT) {
    const int to = h_to(p, h);
    const int s = (p.hin[to] == 1 && p.hout[to] == 1) ? p.outH[to] : -1;
    p.nxt[h] = s;
    p.J[h] = s;
    p.M[h] = h_from(p, h);
  }
}

// one pointer-jumping round: J <- J o J (-1 once a chain ends), M the lowest start vertex over the doubled window
__global__ void __launch_bounds__(MT) clean_jump_kernel(const int *J, const int *M, int *Jn, int *Mn, const int *bnd)
{
  const int B = *bnd;
  for (int h = blockIdx.x * MT + threadIdx.x; h < B; h += gridDim.x * MT) {
    const int j = J[h];
    Jn[h] = j < 0 ? -1 : J[j];
    Mn[h] = j < 0 ? M[h] : min(M[h], M[j]);
  }
}

// every cycle's start (the half-edge from its lowest vertex): its length, and the fill faces of an eligible one
__global__ void __launch_bounds__(MT) clean_loop_kernel(CleanParams p)
{
  const int B = p.res->bnd;
  unsigned int nl = 0, nch = 0;
  for (int h = blockIdx.x * MT + threadIdx.x; h < B; h += gridDim.x * MT) {
    if (p.J[h] < 0) {
      nch++;
      continue;
    }
    const int from = h_from(p, h);
    if (from != p.M[h]) continue;
    nl++;
    int g = h, L = 0;
    do {
      g = p.nxt[g];
      L++;
    } while (g != h && L <= p.maxHole);
    if (g == h && L >= 3 && L <= p.maxHole) {
      p.fcnt[from] = L - 2;
      p.hstart[from] = h;
    }
  }
  if (nl) atomicAdd(&p.res->loops, nl);
  if (nch) atomicAdd(&p.res->chain, nch);
}

// some kept face holds the edge {a, b} (a binary search of the sorted edge keys, then its run)
__device__ bool edge_exists(const CleanParams &p, int a, int b)
{
  const int lo = edge_lower(p, a, b);
  for (int j = lo; j < 3 * p.T && p.ekeyS[j] == p.ekeyS[lo]; j++)
    if (p.alive[p.ecS[j] / 3]) return true;
  return false;
}

// Ear cutting of the loop that starts at vertex v (rule 6): false when no allowed ear remains
__device__ bool ear_cut(const CleanParams &p, int h, int L, int *out)
{
  int r[MAX_HOLE];
  for (int i = 0, g = h; i < L; i++, g = p.nxt[g]) r[i] = h_from(p, g);
  const D3 p0 = P(p, r[0]);
  D3 N = {0.0, 0.0, 0.0};
  for (int i = 1; i + 1 < L; i++) {
    const D3 n = normal3(p0, P(p, r[i]), P(p, r[i + 1]));
    N = {N.x + n.x, N.y + n.y, N.z + n.z};
  }
  int n = L, e = 0;
  while (n > 3) {
    int best = -1;
    double bc = 0.0;
    for (int i = 0; i < n; i++) {
      const D3 pa = P(p, r[i == 0 ? n - 1 : i - 1]), pb = P(p, r[i]), pc = P(p, r[i + 1 == n ? 0 : i + 1]);
      if (!(dot3(normal3(pa, pb, pc), N) > 0.0)) continue;
      if (edge_exists(p, r[i == 0 ? n - 1 : i - 1], r[i + 1 == n ? 0 : i + 1])) continue;
      bool inside = false;
      for (int j = 0; j < n && !inside; j++) {
        const int q = r[j];
        if (q == r[i] || q == r[i == 0 ? n - 1 : i - 1] || q == r[i + 1 == n ? 0 : i + 1]) continue;
        const D3 pq = P(p, q);
        inside = dot3(normal3(pa, pb, pq), N) > 0.0 && dot3(normal3(pb, pc, pq), N) > 0.0 &&
                 dot3(normal3(pc, pa, pq), N) > 0.0;
      }
      if (inside) continue;
      const D3 u = sub3(pa, pb), w = sub3(pc, pb);
      const double cs = dot3(u, w) / sqrt(dot3(u, u) * dot3(w, w));
      if (best < 0 || cs > bc) {
        best = i;
        bc = cs;
      }
    }
    if (best < 0) return false;
    out[3 * e] = r[best == 0 ? n - 1 : best - 1];
    out[3 * e + 1] = r[best];
    out[3 * e + 2] = r[best + 1 == n ? 0 : best + 1];
    e++;
    for (int j = best; j + 1 < n; j++) r[j] = r[j + 1];
    n--;
  }
  if (!(dot3(normal3(P(p, r[0]), P(p, r[1]), P(p, r[2])), N) > 0.0)) return false;
  out[3 * e] = r[0];
  out[3 * e + 1] = r[1];
  out[3 * e + 2] = r[2];
  return true;
}

__global__ void __launch_bounds__(MT) clean_ear_kernel(CleanParams p)
{
  unsigned int nf = 0;
  for (int v = blockIdx.x * MT + threadIdx.x; v < p.V; v += gridDim.x * MT) {
    const int k = p.fcnt[v];
    const bool ok = k > 0 && ear_cut(p, p.hstart[v], k + 2, p.fillS + 3 * (size_t)p.foff[v]);
    p.okc[v] = ok ? k : 0;
    nf += ok;
  }
  if (nf) atomicAdd(&p.res->filled, nf);
}

// ---- the output faces -----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MT) clean_fcount_kernel(CleanParams p)
{
  const int t = blockIdx.x * MT + threadIdx.x;
  counted_cta_count<MT>(t < p.T ? p.alive[t] : 0, p.blockCounts + blockIdx.x);
}

__global__ void __launch_bounds__(MT) clean_fwrite_kernel(CleanParams p)
{
  const int t = blockIdx.x * MT + threadIdx.x;
  const int keep = t < p.T ? p.alive[t] : 0;
  const int at = p.blockOffsets[blockIdx.x] + counted_position<MT>(keep);
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
    const int k = (int)counted_total(p.blockOffsets, p.blockCounts, gridDim.x - 1);
    p.res->kept = k;
    p.res->tris = k;
  }
  if (!keep) return;
  for (int j = 0; j < 3; j++) p.ftri[3 * (size_t)at + j] = p.tin[3 * (size_t)t + j];
}

// the fill faces of the filled loops, by start vertex, after the kept input faces
__global__ void __launch_bounds__(MT) clean_fillcopy_kernel(CleanParams p)
{
  const int kept = p.res->kept;
  for (int v = blockIdx.x * MT + threadIdx.x; v < p.V; v += gridDim.x * MT) {
    if (v == 0) {
      p.res->fill = p.fpos[p.V];
      p.res->tris = kept + p.fpos[p.V];
    }
    const int k = p.okc[v];
    for (int i = 0; i < 3 * k; i++)
      p.ftri[3 * ((size_t)kept + p.fpos[v]) + i] = p.fillS[3 * (size_t)p.foff[v] + i];
  }
}

// ---- rule 7 ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MT) clean_dkey_kernel(CleanParams p, int T)
{
  for (int c = blockIdx.x * MT + threadIdx.x; c < 3 * T; c += gridDim.x * MT) {
    const unsigned long long a = (unsigned int)p.ftri[c], b = (unsigned int)p.ftri[nextc(c)];
    p.dkey[2 * (size_t)c] = (a << 32) | b;
    p.dkey[2 * (size_t)c + 1] = (b << 32) | a;
  }
}

// a vertex's range of sorted directed keys; a directed key held other than twice (an edge of other than two faces)
// fixes its first vertex
__global__ void __launch_bounds__(MT) clean_vrange_kernel(CleanParams p, int n)
{
  for (int i = blockIdx.x * MT + threadIdx.x; i < n; i += gridDim.x * MT) {
    const unsigned long long k = p.dkeyS[i];
    const int a = (int)(k >> 32);
    if (i == 0 || (int)(p.dkeyS[i - 1] >> 32) != a) p.vfirst[a] = i;
    if (i == n - 1 || (int)(p.dkeyS[i + 1] >> 32) != a) p.vend[a] = i + 1;
    if (i > 0 && p.dkeyS[i - 1] == k) continue;
    int j = i + 1;
    while (j < n && p.dkeyS[j] == k) j++;
    if (j - i != 2) p.fixed[a] = 1;
  }
}

// x <- x + f (mean of the distinct neighbours - x), neighbours in ascending id, each sum in that order
__global__ void __launch_bounds__(MT) clean_smooth_kernel(CleanParams p, const double *pos, double *posN, double f)
{
  for (int v = blockIdx.x * MT + threadIdx.x; v < p.V; v += gridDim.x * MT) {
    D3 x = vertex_of(pos, v);
    const int s0 = p.vfirst[v], s1 = p.vend[v];
    if (s1 > s0 && !p.fixed[v]) {
      D3 s = {0.0, 0.0, 0.0};
      int k = 0;
      for (int i = s0; i < s1; i++) {
        if (i > s0 && p.dkeyS[i - 1] == p.dkeyS[i]) continue;
        const D3 q = vertex_of(pos, (int)(p.dkeyS[i] & 0xffffffffu));
        s = {s.x + q.x, s.y + q.y, s.z + q.z};
        k++;
      }
      const double kk = (double)k;
      x = {x.x + f * (s.x / kk - x.x), x.y + f * (s.y / kk - x.y), x.z + f * (s.z / kk - x.z)};
    }
    posN[3 * (size_t)v] = x.x;
    posN[3 * (size_t)v + 1] = x.y;
    posN[3 * (size_t)v + 2] = x.z;
  }
}

// ---- rule 8 ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MT) clean_used_kernel(CleanParams p)
{
  const long long n = 3ll * p.res->tris;
  for (long long c = blockIdx.x * MT + threadIdx.x; c < n; c += (long long)gridDim.x * MT) p.used[p.ftri[c]] = 1;
}

__global__ void __launch_bounds__(MT) clean_vcount_kernel(CleanParams p)
{
  const int x = blockIdx.x * MT + threadIdx.x;
  counted_cta_count<MT>(x < p.V ? p.used[x] : 0, p.blockCounts + blockIdx.x);
}

__global__ void __launch_bounds__(MT) clean_vwrite_kernel(CleanParams p)
{
  const int x = blockIdx.x * MT + threadIdx.x;
  const int u = x < p.V ? p.used[x] : 0;
  const int at = p.blockOffsets[blockIdx.x] + counted_position<MT>(u);
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0)
    p.res->verts = (int)counted_total(p.blockOffsets, p.blockCounts, gridDim.x - 1);
  if (!u) return;
  p.used[x] = at;
  if (at >= p.maxOutV) return;
  for (int d = 0; d < 3; d++) p.outV[3 * (size_t)at + d] = __double2float_rn(p.pos[3 * (size_t)x + d]);
  if (p.outI) p.outI[at] = p.iin[x];
}

__global__ void __launch_bounds__(MT) clean_twrite_kernel(CleanParams p)
{
  const int n = min(p.res->tris, p.maxOutT);
  for (int t = blockIdx.x * MT + threadIdx.x; t < n; t += gridDim.x * MT)
    for (int j = 0; j < 3; j++) p.outT[3 * (size_t)t + j] = p.used[p.ftri[3 * (size_t)t + j]];
}

// the pointer-jumping rounds of rule 6: the smallest r with 2^r > 3 numTriangles
int clean_jump_rounds(int numTriangles) { return radix_bits(3ll * std::max(numTriangles, 1)); }

}  // namespace

int clean_run(const float *vin, const float *iin, int V, const int *tin, int T, int removeDegenerate,
              double longEdgeFactor, int removeNonManifold, int minComponentFaces, double minComponentFraction,
              int maxHoleEdges, int smoothIterations, double lambda, double mu, float *outV, float *outI,
              int maxOutV, int *outT, int maxOutT, cudaStream_t st, void *h_res, double *info, long long *stats)
{
  const int C3 = 3 * T;
  const int nbT = idivup(T, MT), nbC = idivup(C3, MT), nbV = idivup(std::max(V, 1), MT);
  const int nbMax = std::max(nbC, nbV);
  const int vbits = radix_bits(std::max(V, 1));
  const int tiles = idivup(C3, CO_TREE_TILE), groups = idivup(tiles, MT);
  size_t tb[4] = {};
  CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb[0], (int *)nullptr, (int *)nullptr, (int *)nullptr,
                                          (int *)nullptr, T, 0, vbits, st));
  CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb[1], (unsigned long long *)nullptr,
                                          (unsigned long long *)nullptr, (int *)nullptr, (int *)nullptr, C3, 0, 32 + vbits,
                                          st));
  CS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb[2], (int *)nullptr, (int *)nullptr, V + 1, st));
  CS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb[3], (int *)nullptr, (int *)nullptr, nbMax, st));
  size_t tempBytes = 0;
  for (size_t b : tb) tempBytes = std::max(tempBytes, b);

  const size_t T4 = (size_t)T * 4, C4 = (size_t)C3 * 4, V4 = ((size_t)V + 1) * 4;
  Layout L(256);
  const size_t resAt = L.take(sizeof(CleanResult));
  const size_t aliveAt = L.take(T4), dropAt = L.take(T4), parAt = L.take(T4), sizeAt = L.take(T4);
  const size_t k1At = L.take(T4), fvAt = L.take(T4), fvSAt = L.take(T4), fv2SAt = L.take(T4);
  const size_t k2At = L.take((size_t)T * 8);
  const size_t cparAt = L.take(C4), ekAt = L.take(C4 * 2), ekSAt = L.take(C4 * 2), ecAt = L.take(C4),
               ecSAt = L.take(C4);
  const size_t partAt = L.take((size_t)tiles * 24 + 24), groupAt = L.take((size_t)groups * 24 + 24);
  const size_t bflAt = L.take(C4), blAt = L.take(C4), nxtAt = L.take(C4), jAt = L.take(C4), jnAt = L.take(C4),
               mAt = L.take(C4), mnAt = L.take(C4);
  const size_t fansAt = L.take(V4), hinAt = L.take(V4), houtAt = L.take(V4), outHAt = L.take(V4);
  const size_t fcntAt = L.take(V4), foffAt = L.take(V4), hsAt = L.take(V4), okcAt = L.take(V4), fposAt = L.take(V4);
  const size_t fillAt = L.take(C4 * 3), ftriAt = L.take(T4 * 12);
  const size_t vfAt = L.take(V4), veAt = L.take(V4), fixAt = L.take((size_t)V + 1);
  const size_t posAt = L.take((size_t)V * 24), posNAt = L.take((size_t)V * 24), usedAt = L.take(V4);
  const size_t bcAt = L.take((size_t)nbMax * 4), boAt = L.take((size_t)nbMax * 4);
  const size_t tempAt = L.take(tempBytes);
  char *base = nullptr;
  CS_CUDA(cudaMallocAsync((void **)&base, L.bytes, st));
  auto at = [&](size_t off) { return base + off; };
  auto I = [&](size_t off) { return reinterpret_cast<int *>(at(off)); };
  auto U = [&](size_t off) { return reinterpret_cast<unsigned long long *>(at(off)); };

  CleanParams p{};
  p.res = reinterpret_cast<CleanResult *>(at(resAt));
  p.V = V;
  p.T = T;
  p.vin = vin;
  p.iin = iin;
  p.tin = tin;
  p.alive = I(aliveAt);
  p.drop = I(dropAt);
  p.parent = I(parAt);
  p.size = I(sizeAt);
  p.cparent = I(cparAt);
  p.fans = I(fansAt);
  p.k1 = I(k1At);
  p.fv = I(fvAt);
  p.fvS = I(fvSAt);
  p.fv2S = I(fv2SAt);
  p.k2 = U(k2At);
  p.ekey = U(ekAt);
  p.ekeyS = U(ekSAt);
  p.ec = I(ecAt);
  p.ecS = I(ecSAt);
  p.part = reinterpret_cast<double *>(at(partAt));
  p.group = reinterpret_cast<double *>(at(groupAt));
  p.bflag = I(bflAt);
  p.blist = I(blAt);
  p.nxt = I(nxtAt);
  p.J = I(jAt);
  p.Jn = I(jnAt);
  p.M = I(mAt);
  p.Mn = I(mnAt);
  p.hin = I(hinAt);
  p.hout = I(houtAt);
  p.outH = I(outHAt);
  p.fcnt = I(fcntAt);
  p.foff = I(foffAt);
  p.hstart = I(hsAt);
  p.okc = I(okcAt);
  p.fpos = I(fposAt);
  p.fillS = I(fillAt);
  p.ftri = I(ftriAt);
  p.vfirst = I(vfAt);
  p.vend = I(veAt);
  p.fixed = reinterpret_cast<unsigned char *>(at(fixAt));
  p.pos = reinterpret_cast<double *>(at(posAt));
  p.posN = reinterpret_cast<double *>(at(posNAt));
  p.used = I(usedAt);
  p.blockCounts = I(bcAt);
  p.blockOffsets = I(boAt);
  p.minFaces = minComponentFaces;
  p.minFraction = minComponentFraction;
  p.longFactor = longEdgeFactor;
  p.maxHole = maxHoleEdges;
  p.outV = outV;
  p.outI = outI;
  p.outT = outT;
  p.maxOutV = maxOutV;
  p.maxOutT = maxOutT;
  void *temp = at(tempAt);
  CleanResult &R = *static_cast<CleanResult *>(h_res);
  cudaEvent_t *tev = match_timing_events();
  char *dbase = nullptr;

  int status = 0;
  auto readback = [&]() -> int {
    CS_CUDA(cudaMemcpyAsync(h_res, p.res, sizeof(CleanResult), cudaMemcpyDeviceToHost, st));
    CS_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  auto launched = [&](int n) -> int {
    count_launch(n);
    CS_CUDA(cudaGetLastError());
    return 0;
  };
  auto run = [&]() -> int {
    int r;
    if (tev) CS_CUDA(cudaEventRecord(tev[0], st));
    CS_CUDA(cudaMemsetAsync(p.res, 0, sizeof(CleanResult), st));
    mesh_validate_kernel<<<grid_of(T), MT, 0, st>>>(vin, V, tin, T, &p.res->bad);
    if ((r = launched(1)) < 0 || (r = readback()) < 0) return r;
    if (R.bad) {
      status = 2;
      return 0;
    }
    CS_CUDA(cudaMemsetAsync(p.size, 0, T4, st));
    CS_CUDA(cudaMemsetAsync(p.fans, 0, V4, st));
    clean_init_kernel<<<grid_of(std::max(V, C3)), MT, 0, st>>>(p);
    if ((r = launched(1)) < 0) return r;
    clean_edge_key_kernel<<<grid_of(C3), MT, 0, st>>>(p);
    if ((r = launched(1)) < 0) return r;
    CS_CUDA(cub::DeviceRadixSort::SortPairs(temp, tempBytes, p.ekey, p.ekeyS, p.ec, p.ecS, C3, 0, 32 + vbits, st));
    // rule 2 (the sorted keys go to ekey, which is free once the edge keys are sorted)
    if (removeDegenerate) {
      clean_face_key_kernel<<<grid_of(T), MT, 0, st>>>(p);
      if ((r = launched(1)) < 0) return r;
      CS_CUDA(cub::DeviceRadixSort::SortPairs(temp, tempBytes, p.k1, reinterpret_cast<int *>(p.ekey), p.fv, p.fvS, T,
                                              0, vbits, st));
      clean_face_key2_kernel<<<grid_of(T), MT, 0, st>>>(p);
      if ((r = launched(1)) < 0) return r;
      CS_CUDA(cub::DeviceRadixSort::SortPairs(temp, tempBytes, p.k2, p.ekey, p.fvS, p.fv2S, T, 0, 32 + vbits, st));
      clean_duplicate_kernel<<<grid_of(T), MT, 0, st>>>(p);
      if ((r = launched(1)) < 0) return r;
    }
    // rule 3
    if (longEdgeFactor > 0.0) {
      clean_edge_tiles_kernel<<<std::min(tiles, 8192), MT, 0, st>>>(p);
      clean_edge_groups_kernel<<<std::min(groups, 8192), MT, 0, st>>>(p);
      clean_edge_total_kernel<<<1, MT, 0, st>>>(p);
      clean_long_kernel<<<grid_of(T), MT, 0, st>>>(p);
      if ((r = launched(4)) < 0) return r;
    }
    // rule 4
    if (removeNonManifold) {
      CS_CUDA(cudaMemsetAsync(p.drop, 0, T4, st));
      clean_fin_mark_kernel<<<grid_of(C3), MT, 0, st>>>(p);
      clean_fin_drop_kernel<<<grid_of(T), MT, 0, st>>>(p);
      if ((r = launched(2)) < 0) return r;
    }
    // rule 5
    clean_link_kernel<<<grid_of(C3), MT, 0, st>>>(p);
    clean_roots_kernel<<<grid_of(T), MT, 0, st>>>(p);
    clean_count_kernel<<<grid_of(std::max(T, V)), MT, 0, st>>>(p);
    if ((r = launched(3)) < 0) return r;
    if (minComponentFaces > 1 || minComponentFraction > 0.0) {
      clean_small_kernel<<<grid_of(T), MT, 0, st>>>(p);
      if ((r = launched(1)) < 0) return r;
    }
    if (tev) CS_CUDA(cudaEventRecord(tev[1], st));
    // rule 6
    if (maxHoleEdges > 0) {
      CS_CUDA(cudaMemsetAsync(p.bflag, 0, C4, st));
      CS_CUDA(cudaMemsetAsync(p.hin, 0, V4, st));
      CS_CUDA(cudaMemsetAsync(p.hout, 0, V4, st));
      CS_CUDA(cudaMemsetAsync(p.fcnt, 0, V4, st));
      CS_CUDA(cudaMemsetAsync(p.okc, 0, V4, st));
      clean_boundary_kernel<<<grid_of(C3), MT, 0, st>>>(p);
      clean_bcount_kernel<<<nbC, MT, 0, st>>>(p);
      if ((r = launched(2)) < 0) return r;
      CS_CUDA(cub::DeviceScan::ExclusiveSum(temp, tempBytes, p.blockCounts, p.blockOffsets, nbC, st));
      clean_bwrite_kernel<<<nbC, MT, 0, st>>>(p);
      clean_succ_kernel<<<grid_of(C3), MT, 0, st>>>(p);
      if ((r = launched(2)) < 0) return r;
      const int rounds = clean_jump_rounds(T);
      for (int k = 0; k < rounds; k++) {
        clean_jump_kernel<<<grid_of(C3), MT, 0, st>>>(p.J, p.M, p.Jn, p.Mn, &p.res->bnd);
        std::swap(p.J, p.Jn);
        std::swap(p.M, p.Mn);
      }
      clean_loop_kernel<<<grid_of(C3), MT, 0, st>>>(p);
      if ((r = launched(rounds + 1)) < 0) return r;
      CS_CUDA(cub::DeviceScan::ExclusiveSum(temp, tempBytes, p.fcnt, p.foff, V + 1, st));
      clean_ear_kernel<<<grid_of(V), MT, 0, st>>>(p);
      if ((r = launched(1)) < 0) return r;
      CS_CUDA(cub::DeviceScan::ExclusiveSum(temp, tempBytes, p.okc, p.fpos, V + 1, st));
    }
    clean_fcount_kernel<<<nbT, MT, 0, st>>>(p);
    if ((r = launched(1)) < 0) return r;
    CS_CUDA(cub::DeviceScan::ExclusiveSum(temp, tempBytes, p.blockCounts, p.blockOffsets, nbT, st));
    clean_fwrite_kernel<<<nbT, MT, 0, st>>>(p);
    if ((r = launched(1)) < 0) return r;
    if (maxHoleEdges > 0) {
      clean_fillcopy_kernel<<<grid_of(V), MT, 0, st>>>(p);
      if ((r = launched(1)) < 0) return r;
    }
    if (tev) CS_CUDA(cudaEventRecord(tev[2], st));
    // rule 7
    if (smoothIterations > 0) {
      if ((r = readback()) < 0) return r;
      const int Tf = R.tris, D = 6 * Tf;
      size_t sb = 0;
      CS_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, sb, (unsigned long long *)nullptr,
                                             (unsigned long long *)nullptr, D, 0, 32 + vbits, st));
      Layout S(256);
      const size_t dAt = S.take((size_t)D * 8), dSAt = S.take((size_t)D * 8), sAt = S.take(sb);
      CS_CUDA(cudaMallocAsync((void **)&dbase, S.bytes, st));
      p.dkey = reinterpret_cast<unsigned long long *>(dbase + dAt);
      p.dkeyS = reinterpret_cast<unsigned long long *>(dbase + dSAt);
      CS_CUDA(cudaMemsetAsync(p.vfirst, 0, V4, st));
      CS_CUDA(cudaMemsetAsync(p.vend, 0, V4, st));
      CS_CUDA(cudaMemsetAsync(p.fixed, 0, (size_t)V + 1, st));
      clean_dkey_kernel<<<grid_of(3ll * Tf), MT, 0, st>>>(p, Tf);
      if ((r = launched(1)) < 0) return r;
      CS_CUDA(cub::DeviceRadixSort::SortKeys(dbase + sAt, sb, p.dkey, p.dkeyS, D, 0, 32 + vbits, st));
      clean_vrange_kernel<<<grid_of(D), MT, 0, st>>>(p, D);
      if ((r = launched(1)) < 0) return r;
      for (int it = 0; it < smoothIterations; it++) {
        clean_smooth_kernel<<<grid_of(V), MT, 0, st>>>(p, p.pos, p.posN, lambda);
        clean_smooth_kernel<<<grid_of(V), MT, 0, st>>>(p, p.posN, p.pos, mu);
        if ((r = launched(2)) < 0) return r;
      }
    }
    if (tev) CS_CUDA(cudaEventRecord(tev[3], st));
    // rule 8
    CS_CUDA(cudaMemsetAsync(p.used, 0, V4, st));
    clean_used_kernel<<<grid_of(3ll * T), MT, 0, st>>>(p);
    clean_vcount_kernel<<<nbV, MT, 0, st>>>(p);
    if ((r = launched(2)) < 0) return r;
    CS_CUDA(cub::DeviceScan::ExclusiveSum(temp, tempBytes, p.blockCounts, p.blockOffsets, nbV, st));
    clean_vwrite_kernel<<<nbV, MT, 0, st>>>(p);
    clean_twrite_kernel<<<grid_of(3ll * T), MT, 0, st>>>(p);
    if ((r = launched(2)) < 0) return r;
    if ((r = readback()) < 0) return r;
    if (tev) {
      CS_CUDA(cudaEventRecord(tev[4], st));
      static const char *const names[4] = {"rules 2-5", "holes", "smoothing", "output"};
      report_stage_times(tev, names, 4, "clean timing triangles=%d", T);
    }
    return 0;
  };
  const int r = run();
  if (dbase) cudaFreeAsync(dbase, st);
  cudaFreeAsync(base, st);
  if (r < 0) return r;
  const bool out = status != 2;
  const long long Vout = out ? R.verts : 0, Tout = out ? R.tris : 0;
  if (info) {
    info[0] = out ? R.mean : 0.0;
    info[1] = out ? R.sdev : 0.0;
    info[2] = out ? R.thr : 0.0;
  }
  if (stats) {
    const long long s[19] = {T, R.degenerate, R.duplicate, R.longEdge, R.nonManifold, R.small, R.components,
                             R.removed, R.nmVertices, R.loops, R.filled, (long long)R.loops - R.filled, R.chain,
                             R.fill, Vout, Tout, std::min(Vout, (long long)maxOutV),
                             std::min(Tout, (long long)maxOutT), status};
    for (int k = 0; k < 19; k++) stats[k] = (out || k == 0 || k == 18) ? s[k] : 0;
  }
  return (int)Tout;
}

size_t clean_result_bytes() { return sizeof(CleanResult); }

}  // namespace cs
