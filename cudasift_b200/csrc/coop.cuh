// coop.cuh -- the fixed-order machinery of a cooperative solver: bundle adjustment (bundle.cu), rotation averaging
// (rotavg.cu) and global positioning (globalpos.cu) over a sorted incidence list; the MGPCG solves of Poisson meshing
// (mesh.cu) and the energy totals of mesh texturing (texture.cu) take the three-level totals only.  The first three
// sort their incidences (observation or edge end) by item (camera or image) with a stable radix sort; each solver runs
// one cooperative kernel whose phases are separated by grid barriers.  Every floating-point sum has a fixed order that
// depends on the data only, not on the grid or on scheduling:
//   - per item: the sorted incidences are cut into tiles of CO_TILE; a warp sums an item's piece of a tile
//     lane-strided, then by a fixed xor butterfly, and one lane per item adds its pieces in ascending tile order;
//   - totals: a CTA sums a tile of its threads' values by butterflies and its warps in order, or a warp sums a tile of
//     32 lanes' values by a butterfly; the tile partials are then added by warp 0 of every CTA, lane-strided in
//     ascending order and by a butterfly;
//   - three-level totals, for item counts whose tile partials are too many for every CTA to read: tiles of
//     CO_TREE_TILE items, then groups of THREADS tile partials the same way, then the group partials by warp 0 of every
//     CTA (co_tree_tiles, co_tree_groups, co_tree_total).
// No floating-point atomics.  A total is read by every CTA after the grid barrier that follows the writes of its
// partials, so every CTA computes it from the same words by the same instructions, and a branch around a grid barrier
// taken on it is taken alike by every CTA.  That holds only while the partials stay put: a slot read after barrier b
// may be written again only in a phase that follows barrier b + 1 (DESIGN.md, bundle adjustment).
#pragma once

#include "vp_math.cuh"

namespace cs {

constexpr int CO_TILE = 256;         // sorted incidences per item tile
constexpr int CO_TREE_TILE = 2048;   // items per tile of a three-level total

// The K sums of n tile partials (part[tile * stride + j]): warp 0 adds them lane-strided in ascending order, then by a
// fixed xor butterfly; every thread of the CTA receives them.  Every CTA reads the partials after the barrier that
// follows their writes, so a slot read here must not be written again before the next grid barrier.
template <int K>
__device__ __forceinline__ void co_totals(const double *part, int n, int stride, double (&out)[K])
{
  __shared__ double s_tot[K];
  if (threadIdx.x < 32) {
    double v[K];
#pragma unroll
    for (int j = 0; j < K; j++) v[j] = 0.0;
    for (int i = (int)threadIdx.x; i < n; i += 32)
#pragma unroll
      for (int j = 0; j < K; j++) v[j] += part[(size_t)i * stride + j];
    vp_warp_sum(v);
    if (threadIdx.x == 0)
#pragma unroll
      for (int j = 0; j < K; j++) s_tot[j] = v[j];
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < K; j++) out[j] = s_tot[j];
  __syncthreads();                                           // s_tot is read before the next call writes it
}

// A CTA's tile partial of K values (one per thread): warp butterflies, then thread 0 adds the WARPS warps in order.
template <int K, int WARPS>
__device__ __forceinline__ void co_cta_partial(double (&v)[K], double *out)
{
  __shared__ double s_w[WARPS][K];
  vp_warp_sum(v);
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int j = 0; j < K; j++) s_w[threadIdx.x >> 5][j] = v[j];
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int j = 0; j < K; j++) {
      double s = s_w[0][j];
      for (int w = 1; w < WARPS; w++) s += s_w[w][j];
      out[j] = s;
    }
  __syncthreads();
}

// A warp's tile partial of K values (one per lane, a lane per item): a butterfly, lane 0 writes.
template <int K>
__device__ __forceinline__ void co_warp_partial(double (&v)[K], double *out)
{
  vp_warp_sum(v);
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int j = 0; j < K; j++) out[j] = v[j];
}

// Per item i < n (a thread each, tiles of THREADS items per CTA): f(i, v) gives K values for the tile partials at part
// (or nothing with K == 0); v starts at zero.
template <int K, int THREADS, class F>
__device__ __forceinline__ void co_per_item(int n, double *part, F &&f)
{
  for (int base = (int)blockIdx.x * THREADS; base < n; base += (int)gridDim.x * THREADS) {
    const int i = base + (int)threadIdx.x;
    double v[K > 0 ? K : 1];
#pragma unroll
    for (int j = 0; j < (K > 0 ? K : 1); j++) v[j] = 0.0;
    if (i < n) f(i, v);
    if constexpr (K > 0) co_cta_partial<K, THREADS / 32>(v, part + (size_t)(base / THREADS) * K);
  }
}

// Level 1 of a three-level total over n items in CTAs of THREADS threads: every item i < n, tile by tile (tile t: items
// t CO_TREE_TILE + m THREADS + thread), f(i, v) may do any per-item work and adds its K values to v (zero at the start
// of the tile); each tile's partial goes to part[t][K].
template <int K, int THREADS, class F>
__device__ __forceinline__ void co_tree_tiles(int n, double *part, F &&f)
{
  const int tiles = (n + CO_TREE_TILE - 1) / CO_TREE_TILE;
  for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
    double v[K];
#pragma unroll
    for (int j = 0; j < K; j++) v[j] = 0.0;
    for (int m = 0; m < CO_TREE_TILE / THREADS; m++) {
      const int i = t * CO_TREE_TILE + m * THREADS + (int)threadIdx.x;
      if (i < n) f(i, v);
    }
    co_cta_partial<K, THREADS / 32>(v, part + (size_t)t * K);
  }
}

// Level 2, after the grid barrier that follows level 1: group g of THREADS tile partials sums tiles g THREADS + thread
// into group[g][K].
template <int K, int THREADS>
__device__ __forceinline__ void co_tree_groups(int n, const double *part, double *group)
{
  const int tiles = (n + CO_TREE_TILE - 1) / CO_TREE_TILE, groups = (tiles + THREADS - 1) / THREADS;
  for (int g = blockIdx.x; g < groups; g += gridDim.x) {
    double v[K];
    const int t = g * THREADS + (int)threadIdx.x;
#pragma unroll
    for (int j = 0; j < K; j++) v[j] = t < tiles ? part[(size_t)t * K + j] : 0.0;
    co_cta_partial<K, THREADS / 32>(v, group + (size_t)g * K);
  }
}

// Level 3, after the grid barrier that follows level 2: the K totals of the group partials by co_totals.
template <int K, int THREADS>
__device__ __forceinline__ void co_tree_total(int n, const double *group, double (&out)[K])
{
  co_totals<K>(group, ((n + CO_TREE_TILE - 1) / CO_TREE_TILE + THREADS - 1) / THREADS, K, out);
}

// co_per_item over the tracks that have observations: f(k, s, e, v) with [s, e) = [start[k], start[k + 1]) not empty.
template <int K, int THREADS, class F>
__device__ __forceinline__ void co_per_track(const int *start, int numTracks, double *part, F &&f)
{
  co_per_item<K, THREADS>(numTracks, part, [&](int k, double *v) {
    const int s = start[k], e = start[k + 1];
    if (e > s) f(k, s, e, v);
  });
}

// Every item's range [start, end) of the n sorted keys (items[a].start, items[a].end; an item without a key keeps
// its zeroed range).
template <class Item>
__device__ __forceinline__ void co_ranges(const int *keysS, int n, Item *items, int tid, int nthreads)
{
  for (int i = tid; i < n; i += nthreads) {
    const int a = keysS[i];
    if (i == 0 || keysS[i - 1] != a) items[a].start = i;
    if (i == n - 1 || keysS[i + 1] != a) items[a].end = i + 1;
  }
}

// The item pieces of NV values per incidence (f(order[i], a, v) for sorted incidence i of item a) at offset OFF of
// pieces of PV values: a warp per tile of CO_TILE sorted incidences, each item's piece summed lane-strided and by a
// butterfly, stored at piece index tile + item (unique: an item's tiles follow the previous item's last one).
template <int NV, int OFF, int PV, int THREADS, class Item, class F>
__device__ __forceinline__ void co_pieces(const int *keysS, const int *order, double *pieces, int n, const Item *items,
                                          F &&f)
{
  const int lane = threadIdx.x & 31;
  const int numWarps = (int)gridDim.x * (THREADS / 32), numTiles = (n + CO_TILE - 1) / CO_TILE;
  for (int t = (int)((blockIdx.x * THREADS + threadIdx.x) >> 5); t < numTiles; t += numWarps) {
    const int t1 = min(n, (t + 1) * CO_TILE);
    for (int s = t * CO_TILE; s < t1;) {
      const int a = keysS[s];
      const int e = min(t1, items[a].end);
      double acc[NV];
#pragma unroll
      for (int j = 0; j < NV; j++) acc[j] = 0.0;
      for (int i = s + lane; i < e; i += 32) {
        double v[NV];
        f(order[i], a, v);
#pragma unroll
        for (int j = 0; j < NV; j++) acc[j] += v[j];
      }
      vp_warp_sum(acc);
      if (lane == 0)
#pragma unroll
        for (int j = 0; j < NV; j++) pieces[(size_t)(t + a) * PV + OFF + j] = acc[j];
      s = e;
    }
  }
}

// The sum of item a's pieces (NV values at OFF of PV) in ascending tile order.
template <int NV, int OFF, int PV, class Item>
__device__ __forceinline__ void co_gather(const double *pieces, int a, const Item &c, double (&v)[NV])
{
#pragma unroll
  for (int j = 0; j < NV; j++) v[j] = 0.0;
  if (c.end > c.start)
    for (int t = c.start / CO_TILE; t <= (c.end - 1) / CO_TILE; t++)
#pragma unroll
      for (int j = 0; j < NV; j++) v[j] += pieces[(size_t)(t + a) * PV + OFF + j];
}

// The count kernel's work for thread k of a track list (P: cnt, numTracks, res->stats) whose track k has used(k,
// invalid) used observations (-1: malformed; invalid: its members that fail tr_member): cnt[k] the count when at least
// 2, else 0 (cnt[numTracks] = 0 for the scan), and the integer statistics stats[0..4]: well-formed tracks, malformed
// tracks, invalid members, used observations and participating tracks.
template <class P, class U>
__device__ __forceinline__ void co_count(const P &p, int k, U &&used)
{
  if (k == 0) p.cnt[p.numTracks] = 0;
  if (k >= p.numTracks) return;
  int invalid = 0;
  const int n = used(k, invalid);
  unsigned long long *st = p.res->stats;
  if (n < 0) {
    atomicAdd(&st[1], 1ull);
    p.cnt[k] = 0;
    return;
  }
  atomicAdd(&st[0], 1ull);
  if (invalid) atomicAdd(&st[2], (unsigned long long)invalid);
  p.cnt[k] = n >= 2 ? n : 0;
  if (n >= 2) {
    atomicAdd(&st[3], (unsigned long long)n);
    atomicAdd(&st[4], 1ull);
  }
}

}  // namespace cs
