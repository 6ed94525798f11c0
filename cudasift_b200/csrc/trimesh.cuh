// trimesh.cuh -- the triangle-mesh helpers of mesh simplification (simplify.cu), mesh texturing (texture.cu) and seam
// levelling (seams.cu): the float64 vectors, the vertex load, the tie order s(id), the input check of rule 1, the edge
// keys and adjacency, the lower-vertex edge rule and the launch shape.
//
// Include it only from units compiled with -fmad=false (build.py's UNIT_FLAGS).  Its float64 expressions must round
// once per product and sum, in the order written, as tests/simplify_oracle.py and tests/texture_oracle.py compute
// them; in a unit that lets nvcc contract a product and a sum into an fma, the same source gives other bits.
#pragma once

#include "common.cuh"

namespace cs {

namespace {

constexpr int MT = 256;                       // threads per CTA of every simplify and texture kernel

struct D3 {
  double x, y, z;
};
__device__ __forceinline__ D3 sub3(D3 a, D3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ D3 cross3(D3 a, D3 b)
{
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
__device__ __forceinline__ double dot3(D3 a, D3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ D3 normal3(D3 p0, D3 p1, D3 p2) { return cross3(sub3(p1, p0), sub3(p2, p0)); }

// vertex v of a [V][3] array of float or double
template <class T>
__device__ __forceinline__ D3 vertex_of(const T *xyz, int v)
{
  return {(double)xyz[3 * (size_t)v], (double)xyz[3 * (size_t)v + 1], (double)xyz[3 * (size_t)v + 2]};
}

// The tie order s(id): simplification's key order for equal errors (rule 5 of cs_simplify_mesh) and texturing's
// colouring priority.  A bijection of the 32-bit ids (an odd multiplier mod 2^32, then an invertible xorshift), so keys
// stay unique while equal errors are not ranked in raster order.
__device__ __forceinline__ unsigned int tie_of(unsigned int id)
{
  const unsigned int m = id * 0x9E3779B1u;
  return m ^ (m >> 16);
}

// Rule 1 of cs_simplify_mesh and cs_texture_mesh: *bad |= 1 when a triangle has an index outside [0, V), repeats a
// vertex, or has a corner with a non-finite coordinate.
__global__ void __launch_bounds__(MT) mesh_validate_kernel(const float *vin, int V, const int *tin, int T,
                                                          unsigned int *bad)
{
  for (int t = blockIdx.x * MT + threadIdx.x; t < T; t += gridDim.x * MT) {
    const int a = tin[3 * (size_t)t], b = tin[3 * (size_t)t + 1], c = tin[3 * (size_t)t + 2];
    bool fail = a < 0 || a >= V || b < 0 || b >= V || c < 0 || c >= V || a == b || b == c || a == c;
    for (int j = 0; j < 3 && !fail; j++) {
      const int w = tin[3 * (size_t)t + j];
      for (int d = 0; d < 3; d++) fail = fail || !isfinite(vin[3 * (size_t)w + d]);
    }
    if (fail) atomicOr(bad, 1u);
  }
}

// Rule 1 of cs_texture_mesh, the edge keys of texturing (texture.cu) and seam levelling (seams.cu): corner c = 3t + k
// starts the undirected edge from corner k to corner k + 1 mod 3, keyed (min << 32) | max of its two vertices.
__device__ __forceinline__ unsigned long long edge_key_of(const int *tin, int c)
{
  const int t = c / 3, k = c - 3 * t;
  const unsigned int a = tin[c], b = tin[3 * t + (k + 1) % 3];
  return ((unsigned long long)min(a, b) << 32) | max(a, b);
}

// Two faces are adjacent across an edge when exactly two corners hold its key: at position i of the n sorted keys
// (keysS, their corners valsS), a run of exactly two equal keys joins its two faces in nbr [3T].
__device__ __forceinline__ void edge_pair_join(const unsigned long long *keysS, const int *valsS, int *nbr, int i, int n)
{
  const unsigned long long k = keysS[i];
  if ((i > 0 && keysS[i - 1] == k) || keysS[i + 1] != k || (i + 2 < n && keysS[i + 2] == k)) return;
  const int c1 = valsS[i], c2 = valsS[i + 1];
  nbr[c1] = c2 / 3;
  nbr[c2] = c1 / 3;
}

// The lower-vertex edge rule of texturing's key rasters (rule 2 of cs_texture_mesh, rule 7 of
// cs_level_texture_seams): edge k runs corner k -> k + 1; it is evaluated from its lower vertex id P to the higher Q,
// then signed by s = sign(doubled area) and negated when corner k holds the higher id, so the two faces of an edge see
// exactly opposite values and no sample centre on a shared edge is missed.
struct EdgeFns {
  int P[3];
  double du[3], dv[3], sg[3];
};
__device__ __forceinline__ void edge_fns_of(const int (&id)[3], const double (&u)[3], const double (&v)[3], double s,
                                            EdgeFns &e)
{
  for (int k = 0; k < 3; k++) {
    const int a = k, b = (k + 1) % 3;
    const bool lo = id[a] < id[b];
    e.P[k] = lo ? a : b;
    const int Q = lo ? b : a;
    e.du[k] = u[Q] - u[e.P[k]];
    e.dv[k] = v[Q] - v[e.P[k]];
    e.sg[k] = lo ? s : -s;
  }
}
// w_k at the sample centre (x, y)
__device__ __forceinline__ double edge_fn(const EdgeFns &e, const double (&u)[3], const double (&v)[3], int k, double x,
                                          double y)
{
  return e.sg[k] * (e.du[k] * (y - v[e.P[k]]) - e.dv[k] * (x - u[e.P[k]]));
}

// CTAs of a grid-stride launch over n items: one per MT items, at least 1, at most 8192.
int grid_of(long long n) { return (int)std::max(1ll, std::min((n + MT - 1) / MT, 8192ll)); }

}  // namespace

}  // namespace cs
