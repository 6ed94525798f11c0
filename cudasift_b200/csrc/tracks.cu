// tracks.cu -- feature tracks over the pair lists of many image pairs (cs_build_tracks).
//
// Feature f of image a has the global id g = base[a] + f.  The kernels, in order (DESIGN section 4):
//   init      parent[g] = g, value[g] = g, the matched and conflict bytes and the statistics cleared
//   hook      one thread per pair of every list: validate, mark both endpoints matched, join the two trees (uf_link,
//             the union-find of common.cuh)
//   compress  label[g] = uf_find(g), the root, which is the component's smallest id
//   sort      (label, g) pairs of all N features, stably by label over ceil(log2 N) bits (cub::DeviceRadixSort): every
//             component is one run, in ascending label, its members in ascending g
//   mark      per run: its first and end positions, and whether two adjacent members share an image
//   reduce    per tile of positions: the kept runs and their members, and the statistics
//   scan      the tile totals (one CTA): track count T and member count M, d_offsets[T] = M
//   heads     per kept run: its track index and first member, d_offsets
//   members   per position: d_members and d_trackOf
// Nothing depends on the order of the atomics: the labels are component minima, and everything after them is a
// function of the sorted (label, g) sequence.
#include <cub/cub.cuh>

#include <cstring>
#include <vector>

#include "common.cuh"

namespace cs {

namespace {

constexpr int TK_THREADS = 256;
constexpr int TK_ITEMS = 8;
constexpr int TK_TILE = TK_THREADS * TK_ITEMS;   // sorted positions per CTA of the reduce and heads kernels
constexpr int TK_SCAN_THREADS = 512;              // the one-CTA tile scan (at 1024 threads its scan spills)

// A list with pairs, as the hook kernel reads it: its global-id bases and sizes, and its first CTA.
struct TkList {
  const int2 *pairs;
  int n;
  int base1, size1, base2, size2;
  int cta0;
};

// Per-feature and per-tile scratch of a call (tracks_scratch places it).
struct TkBufs {
  int *keys[2], *vals[2];     // the sort's double buffers: keys[0] = label, vals[0] = g; keys[1] = parent first
  int *trackIdx, *trackOff;   // indexed by label: the run's track (-1: not kept) and its first member
  unsigned char *matched, *conf;
  int2 *tiles;                // per tile: (kept runs, their members), then the exclusive prefix
  const int *bases;           // [numImages] global id of each image's first feature
  const TkList *lists;
  unsigned long long *stats;  // the eight statistics of cs_build_tracks
  void *sortTemp; size_t sortBytes;
};

struct SegSums {
  int cnt, mem, matched, comps, conflict, shortc;
  __device__ SegSums operator+(const SegSums &o) const
  {
    return {cnt + o.cnt, mem + o.mem, matched + o.matched, comps + o.comps, conflict + o.conflict, shortc + o.shortc};
  }
};
struct Int2Sum {
  __device__ int2 operator()(const int2 &a, const int2 &b) const { return make_int2(a.x + b.x, a.y + b.y); }
};

__device__ __forceinline__ long long thread_index() { return (long long)blockIdx.x * blockDim.x + threadIdx.x; }

// The image of global id g: the largest a with bases[a] <= g (empty images share their base with the next one).
__device__ __forceinline__ int image_of(const int *__restrict__ bases, int numImages, int g)
{
  int lo = 0, hi = numImages - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (bases[mid] <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(TK_THREADS) tracks_init_kernel(TkBufs b, int N)
{
  const long long g = thread_index();
  if (g < 8) b.stats[g] = 0;
  if (g >= N) return;
  b.keys[1][g] = (int)g;      // parent
  b.vals[0][g] = (int)g;
  b.matched[g] = 0;
  b.conf[g] = 0;
}

__global__ void __launch_bounds__(TK_THREADS) tracks_hook_kernel(TkBufs b, int numLists)
{
  const TkList L = b.lists[table_find(b.lists, numLists, &TkList::cta0, (int)blockIdx.x)];
  const int k = ((int)blockIdx.x - L.cta0) * TK_THREADS + (int)threadIdx.x;
  const bool active = k < L.n;
  const int2 p = active ? L.pairs[k] : make_int2(-1, -1);
  const bool ok = active && (unsigned)p.x < (unsigned)L.size1 && (unsigned)p.y < (unsigned)L.size2;
  // every warp of the CTA is whole and converged here
  const unsigned vb = __ballot_sync(0xffffffffu, ok), ib = __ballot_sync(0xffffffffu, active && !ok);
  if ((threadIdx.x & 31) == 0) {
    if (vb) atomicAdd(&b.stats[0], (unsigned long long)__popc(vb));
    if (ib) atomicAdd(&b.stats[1], (unsigned long long)__popc(ib));
  }
  if (!ok) return;
  const int u = L.base1 + p.x, v = L.base2 + p.y;
  b.matched[u] = 1;
  b.matched[v] = 1;
  uf_link(b.keys[1], u, v);   // keys[1] holds parent until the sort
}

// After every hook: the label of every feature.  The halving stores go to parent only, so each label is the root.
__global__ void __launch_bounds__(TK_THREADS) tracks_compress_kernel(TkBufs b, int N)
{
  const long long g = thread_index();
  if (g < N) b.keys[0][g] = uf_find(b.keys[1], (int)g);
}

// Over the sorted positions (keys / vals the sort's output): the run of label L spans [start[L], end[L]).
__global__ void __launch_bounds__(TK_THREADS) tracks_mark_kernel(const int *__restrict__ keys,
                                                                 const int *__restrict__ vals, int *start, int *end,
                                                                 unsigned char *conf, const int *__restrict__ bases,
                                                                 int numImages, int N)
{
  const long long k = thread_index();
  if (k >= N) return;
  const int L = keys[k];
  const bool head = k == 0 || keys[k - 1] != L;
  if (head) start[L] = (int)k;
  if (k == N - 1 || keys[k + 1] != L) end[L] = (int)k + 1;
  if (!head && image_of(bases, numImages, vals[k]) == image_of(bases, numImages, vals[k - 1])) conf[L] = 1;
}

// Position k's part of the sums: at the head of a matched run, that run.
__device__ __forceinline__ SegSums run_at(long long k, int N, const int *__restrict__ keys, const int *__restrict__ start,
                                          const int *__restrict__ end, const unsigned char *__restrict__ matched,
                                          const unsigned char *__restrict__ conf, int minLength, bool drop)
{
  SegSums s{0, 0, 0, 0, 0, 0};
  if (k >= N) return s;
  const int L = keys[k];
  if (start[L] != k || !matched[L]) return s;
  const int size = end[L] - (int)k;
  const bool isShort = size < minLength, conflict = conf[L] != 0;
  const bool kept = !isShort && !(drop && conflict);
  s.cnt = kept;
  s.mem = kept ? size : 0;
  s.matched = size;
  s.comps = 1;
  s.conflict = !isShort && conflict;
  s.shortc = isShort;
  return s;
}

__global__ void __launch_bounds__(TK_THREADS) tracks_reduce_kernel(TkBufs b, const int *__restrict__ keys,
                                                                   const int *__restrict__ start,
                                                                   const int *__restrict__ end, int N, int minLength,
                                                                   int drop)
{
  using Reduce = cub::BlockReduce<SegSums, TK_THREADS>;
  __shared__ typename Reduce::TempStorage tmp;
  const long long k0 = (long long)blockIdx.x * TK_TILE + (long long)threadIdx.x * TK_ITEMS;
  SegSums s{0, 0, 0, 0, 0, 0};
  for (int i = 0; i < TK_ITEMS; i++) s = s + run_at(k0 + i, N, keys, start, end, b.matched, b.conf, minLength, drop);
  const SegSums t = Reduce(tmp).Sum(s);
  if (threadIdx.x == 0) {
    b.tiles[blockIdx.x] = make_int2(t.cnt, t.mem);
    if (t.matched) atomicAdd(&b.stats[2], (unsigned long long)t.matched);
    if (t.comps) atomicAdd(&b.stats[3], (unsigned long long)t.comps);
    if (t.conflict) atomicAdd(&b.stats[4], (unsigned long long)t.conflict);
    if (t.shortc) atomicAdd(&b.stats[5], (unsigned long long)t.shortc);
  }
}

// One CTA: the exclusive prefix of the tile totals in place, T and M, and d_offsets[T] = M when T <= maxTracks.
__global__ void __launch_bounds__(TK_SCAN_THREADS) tracks_scan_kernel(TkBufs b, int numTiles, int *offsets,
                                                                      int maxTracks)
{
  using Scan = cub::BlockScan<int2, TK_SCAN_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  int2 carry = make_int2(0, 0);
  for (int t0 = 0; t0 < numTiles; t0 += TK_SCAN_THREADS) {
    const int t = t0 + (int)threadIdx.x;
    const int2 v = t < numTiles ? b.tiles[t] : make_int2(0, 0);
    int2 x, total;
    Scan(tmp).ExclusiveScan(v, x, make_int2(0, 0), Int2Sum(), total);
    if (t < numTiles) b.tiles[t] = make_int2(carry.x + x.x, carry.y + x.y);
    carry = make_int2(carry.x + total.x, carry.y + total.y);
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    b.stats[6] = (unsigned long long)carry.x;
    b.stats[7] = (unsigned long long)carry.y;
    if (offsets && carry.x <= maxTracks) offsets[carry.x] = carry.y;
  }
}

// Per kept run: its track index and first member (trackIdx / trackOff at its label) and d_offsets; -1 for a matched run
// that is not kept.
__global__ void __launch_bounds__(TK_THREADS) tracks_heads_kernel(TkBufs b, const int *__restrict__ keys,
                                                                  const int *__restrict__ start,
                                                                  const int *__restrict__ end, int N, int minLength,
                                                                  int drop, int *offsets, int maxTracks)
{
  using Scan = cub::BlockScan<int2, TK_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  const long long k0 = (long long)blockIdx.x * TK_TILE + (long long)threadIdx.x * TK_ITEMS;
  SegSums s[TK_ITEMS];
  int2 sum = make_int2(0, 0);
  for (int i = 0; i < TK_ITEMS; i++) {
    s[i] = run_at(k0 + i, N, keys, start, end, b.matched, b.conf, minLength, drop);
    sum.x += s[i].cnt;
    sum.y += s[i].mem;
  }
  int2 x;
  Scan(tmp).ExclusiveScan(sum, x, make_int2(0, 0), Int2Sum());
  const int2 base = b.tiles[blockIdx.x];
  int t = base.x + x.x, off = base.y + x.y;
  for (int i = 0; i < TK_ITEMS; i++) {
    if (!s[i].comps) continue;
    const int L = keys[k0 + i];
    if (s[i].cnt) {
      b.trackIdx[L] = t;
      b.trackOff[L] = off;
      if (offsets && t <= maxTracks) offsets[t] = off;
      t += 1;
      off += s[i].mem;
    } else {
      b.trackIdx[L] = -1;
    }
  }
}

__global__ void __launch_bounds__(TK_THREADS) tracks_members_kernel(TkBufs b, const int *__restrict__ keys,
                                                                    const int *__restrict__ vals,
                                                                    const int *__restrict__ start, int numImages, int N,
                                                                    int *trackOf, int2 *members, int maxMembers)
{
  const long long k = thread_index();
  if (k >= N) return;
  const int g = vals[k], L = keys[k];
  const int t = b.matched[g] ? b.trackIdx[L] : -1;
  if (trackOf) trackOf[g] = t;
  if (t < 0) return;
  const int pos = b.trackOff[L] + ((int)k - start[L]);
  if (pos < maxMembers) {
    const int a = image_of(b.bases, numImages, g);
    members[pos] = make_int2(a, g - b.bases[a]);
  }
}

int grid_of(long long n, int per) { return (int)((n + per - 1) / per > 0 ? (n + per - 1) / per : 1); }

}  // namespace

// The scratch of a call (header: cs_build_tracks): the statistics, the image bases and the list table, then per tile
// its totals, per feature six ints and two bytes, then the sort's temporary storage.  With base == nullptr only the
// size is computed (tempBytes from cub).
static size_t tracks_layout(char *base, int N, int numImages, int numTables, TkBufs *b, size_t tempBytes)
{
  Layout L(256);
  auto take = [&](size_t bytes) { const size_t at = L.take(bytes); return base ? base + at : nullptr; };
  b->stats = reinterpret_cast<unsigned long long *>(take(8 * sizeof(unsigned long long)));
  b->bases = reinterpret_cast<const int *>(take((size_t)numImages * sizeof(int)));
  b->lists = reinterpret_cast<const TkList *>(take((size_t)numTables * sizeof(TkList)));
  b->tiles = reinterpret_cast<int2 *>(take((size_t)grid_of(N, TK_TILE) * sizeof(int2)));
  for (int k = 0; k < 2; k++) b->keys[k] = reinterpret_cast<int *>(take((size_t)N * sizeof(int)));
  for (int k = 0; k < 2; k++) b->vals[k] = reinterpret_cast<int *>(take((size_t)N * sizeof(int)));
  b->trackIdx = reinterpret_cast<int *>(take((size_t)N * sizeof(int)));
  b->trackOff = reinterpret_cast<int *>(take((size_t)N * sizeof(int)));
  b->matched = reinterpret_cast<unsigned char *>(take((size_t)N));
  b->conf = reinterpret_cast<unsigned char *>(take((size_t)N));
  b->sortTemp = take(tempBytes);
  b->sortBytes = tempBytes;
  return L.bytes;
}

int tracks_enqueue(DeviceCtx &c, const int *imageSizes, int numImages, const cs_track_list *lists, int numLists,
                   int minLength, bool drop, int *trackOf, int *offsets, int maxTracks, int *members, int maxMembers)
{
  // host tables: the image bases and the lists with pairs
  int N = 0;
  std::vector<int> bases((size_t)numImages);
  for (int a = 0; a < numImages; a++) { bases[a] = N; N += imageSizes[a]; }
  std::vector<TkList> table;
  int ctas = 0;
  for (int p = 0; p < numLists; p++) {
    const cs_track_list &l = lists[p];
    if (l.numPairs == 0) continue;
    table.push_back(TkList{reinterpret_cast<const int2 *>(l.pairs), l.numPairs, bases[l.image1],
                           imageSizes[l.image1], bases[l.image2], imageSizes[l.image2], ctas});
    ctas += idivup(l.numPairs, TK_THREADS);
  }
  const int numTables = (int)table.size();
  const int bits = N > 1 ? 32 - __builtin_clz((unsigned)(N - 1)) : 1;   // ceil(log2 N): every label is < 2^bits

  TkBufs b;
  size_t tempBytes = 0;
  {
    cub::DoubleBuffer<int> k(nullptr, nullptr), v(nullptr, nullptr);
    CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tempBytes, k, v, N, 0, bits, c.stream));
  }
  const size_t bytes = tracks_layout(nullptr, N, numImages, numTables, &b, tempBytes);
  int r = c.tracks.grow(bytes);
  if (r < 0) return r;
  tracks_layout(c.tracks.as<char>(), N, numImages, numTables, &b, tempBytes);

  // the bases and the list table go up in one copy from pinned memory (the previous call ended in a synchronize)
  const size_t tableOff = reinterpret_cast<const char *>(b.lists) - reinterpret_cast<const char *>(b.bases);
  const size_t up = tableOff + (size_t)numTables * sizeof(TkList);
  if ((r = c.h_tracks.grow(8 * sizeof(unsigned long long) + up)) < 0) return r;
  char *h = c.h_tracks.as<char>() + 8 * sizeof(unsigned long long);
  if (numImages) memcpy(h, bases.data(), (size_t)numImages * sizeof(int));
  if (numTables) memcpy(h + tableOff, table.data(), (size_t)numTables * sizeof(TkList));
  CS_CUDA(cudaMemcpyAsync(const_cast<int *>(b.bases), h, up, cudaMemcpyHostToDevice, c.stream));

  const cudaStream_t st = c.stream;
  const int gN = grid_of(N, TK_THREADS), tiles = grid_of(N, TK_TILE);
  tracks_init_kernel<<<gN, TK_THREADS, 0, st>>>(b, N);
  tracks_hook_kernel<<<ctas, TK_THREADS, 0, st>>>(b, numTables);
  tracks_compress_kernel<<<gN, TK_THREADS, 0, st>>>(b, N);
  count_launch(3);
  CS_CUDA(cudaGetLastError());
  cub::DoubleBuffer<int> keys(b.keys[0], b.keys[1]), vals(b.vals[0], b.vals[1]);
  if (N > 0) CS_CUDA(cub::DeviceRadixSort::SortPairs(b.sortTemp, tempBytes, keys, vals, N, 0, bits, st));
  // the run bounds reuse the sort's spare buffers
  const int *K = keys.Current(), *V = vals.Current();
  int *start = keys.Alternate(), *end = vals.Alternate();
  const int dr = drop ? 1 : 0;
  tracks_mark_kernel<<<gN, TK_THREADS, 0, st>>>(K, V, start, end, b.conf, b.bases, numImages, N);
  tracks_reduce_kernel<<<tiles, TK_THREADS, 0, st>>>(b, K, start, end, N, minLength, dr);
  tracks_scan_kernel<<<1, TK_SCAN_THREADS, 0, st>>>(b, N > 0 ? tiles : 0, offsets, maxTracks);
  tracks_heads_kernel<<<tiles, TK_THREADS, 0, st>>>(b, K, start, end, N, minLength, dr, offsets, maxTracks);
  tracks_members_kernel<<<gN, TK_THREADS, 0, st>>>(b, K, V, start, numImages, N, trackOf,
                                                   reinterpret_cast<int2 *>(members), maxMembers);
  count_launch(5);
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaMemcpyAsync(c.h_tracks.p, b.stats, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  return 0;
}

}  // namespace cs
