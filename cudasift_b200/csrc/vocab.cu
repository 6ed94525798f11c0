// vocab.cu -- visual vocabulary and image retrieval (cs_vocab_assign, cs_vocab_train, cs_retrieve_pairs).
//
// Assignment: the word of a descriptor is j1 of cs_match_knn2 against the vocabulary, so it runs the batched knn waves
// of match_tc.cu (knn_batch_enqueue) over the jobs (set a, vocabulary); each wave's last step copies the neighbour
// lists' j1 (and for training the best score) to the global feature ids of its sets.
// Training (spherical k-means, Lloyd iterations): assign, compare with the previous assignment (fixed-tile partials),
// then a stable radix sort of (word + 1, global id), the run bounds per word, and one 128-thread CTA per word that sums
// its members per component in float64 in ascending global id.
// Retrieval (tf-idf): a radix sort of (image, word) keys and its runs (the postings), df and the image bounds, idf per
// word, one warp per image for the norm and the fixed-point weights q, a stable sort by word (the inverted file), then
// per wave of queries the integer scoring scatter and a top-k select, and at the end a sort and unique pass of pairs.
// Every score is an exact int64 sum, so the order of the 64-bit atomics does not reach any output.
#include <cub/cub.cuh>

#include <cmath>
#include <cstddef>
#include <vector>

#include "common.cuh"
#include "vp_math.cuh"

namespace cs {

namespace {

// ------------------------------------------------------------------------------ shared pieces
// A non-empty set of a call and the global id of its first feature (table_find on base).
struct VbSet {
  const SiftPoint *pts;
  int base;
};
__device__ __forceinline__ const float *vb_desc(const VbSet *__restrict__ sets, int numSets, int g)
{
  const VbSet &s = sets[table_find(sets, numSets, &VbSet::base, g)];
  return s.pts[g - s.base].data;
}

constexpr unsigned long long GOLDEN = 0x9E3779B97F4A7C15ull;

int key_bits(unsigned long long maxKey)
{
  int b = 1;
  while (b < 64 && (maxKey >> b) != 0) b++;
  return b;
}

// ------------------------------------------------------------------------------ assignment
// The fifth launch of an assignment wave: row r of the wave's lists is feature base + r.
__global__ void vb_words_kernel(const int2 *__restrict__ idx, const float2 *__restrict__ score, int rows,
                                int *__restrict__ wordOf, float *__restrict__ best)
{
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  wordOf[r] = idx[r].x;
  if (best) best[r] = score[r].x;
}

}  // namespace

int vocab_assign_enqueue(DeviceCtx &c, const cs_match_set *sets, int numSets, const void *vocab, int numWords,
                         int *wordOf, float *best, VocabAssign &va)
{
  va.sets.assign(sets, sets + numSets);
  va.sets.push_back(cs_match_set{vocab, numWords});
  va.jobs.resize(numSets);
  va.base.resize(numSets);
  long long base = 0;
  for (int a = 0; a < numSets; a++) {
    va.jobs[a] = cs_match_job{a, numSets, nullptr, 0};
    va.base[a] = (int)base;
    base += sets[a].n;
  }
  va.out.assign(numSets, RatioBatchOut{});
  va.waves = 0;
  return knn_batch_enqueue(c, va.sets.data(), numSets + 1, va.jobs.data(), numSets, false, va.out.data(), "vocab-assign", "words",
                           [&](const KnnWave &w) {
                             const int b = va.base[w.jobs[0]];
                             vb_words_kernel<<<idivup(w.rows, 256), 256, 0, c.stream>>>(w.idx, w.score, w.rows,
                                                                                      wordOf + b, best ? best + b : nullptr);
                             count_launch();
                             CS_CUDA(cudaGetLastError());
                             va.waves++;
                             return 0;
                           });
}

void vocab_assign_stats(const VocabAssign &va, unsigned long long st[5])
{
  for (int k = 0; k < 5; k++) st[k] = 0;
  for (size_t a = 0; a < va.out.size(); a++) {
    const RatioBatchOut &o = va.out[a];
    if (va.sets[a].n == 0 || va.sets.back().n == 0) continue;
    st[0] += o.counters[0][1];
    st[1] += o.counters[0][2];
    st[2] += o.counters[0][0];
    st[3] += (*o.bad1 | *o.bad2) ? 1 : 0;
  }
  st[4] = (unsigned long long)va.waves;
}

// ------------------------------------------------------------------------------ training
namespace {

constexpr int VB_THREADS = 256;
constexpr int VB_CHUNK = 4;                       // consecutive features per thread of the compare kernel
constexpr int VB_TILE = VB_THREADS * VB_CHUNK;    // features per partial

struct VbPartial {
  double sum;                   // best scores of the assigned features of the tile
  unsigned int changed, assigned;
};

// Per tile of VB_TILE features: thread t sums the best scores of the assigned features among tile + 4t .. 4t + 3 in
// that order (float64, from 0), then the tree s = 128, 64, .., 1: x[t] += x[t + s].  The changed and assigned counts are
// integers.  Also the previous assignment is replaced and the sort's (word + 1, global id) pairs are written.
__global__ void __launch_bounds__(VB_THREADS)
vb_compare_kernel(const int *__restrict__ cur, int *__restrict__ prev, const float *__restrict__ best, int M, int first,
                  VbPartial *__restrict__ part, unsigned int *__restrict__ keys, int *__restrict__ vals)
{
  __shared__ double s_sum[VB_THREADS];
  __shared__ unsigned int s_changed, s_assigned;
  const int t = threadIdx.x;
  if (t == 0) { s_changed = 0; s_assigned = 0; }
  const int i0 = blockIdx.x * VB_TILE + VB_CHUNK * t;
  double s = 0.0;
  unsigned int ch = 0, as = 0;
#pragma unroll
  for (int e = 0; e < VB_CHUNK; e++) {
    const int i = i0 + e;
    if (i < M) {
      const int w = cur[i];
      if (w >= 0) { s = __dadd_rn(s, (double)best[i]); as++; }
      if (first || w != prev[i]) ch++;
      prev[i] = w;
      keys[i] = (unsigned int)(w + 1);
      vals[i] = i;
    }
  }
  s_sum[t] = s;
  __syncthreads();
  atomicAdd(&s_changed, ch);
  atomicAdd(&s_assigned, as);
  for (int o = VB_THREADS / 2; o > 0; o >>= 1) {
    if (t < o) s_sum[t] = __dadd_rn(s_sum[t], s_sum[t + o]);
    __syncthreads();
  }
  if (t == 0) part[blockIdx.x] = VbPartial{s_sum[0], s_changed, s_assigned};
}

// The members of word k are the sorted positions [start[k], end[k]) (both 0 for a word without members).
__global__ void vb_bounds_kernel(const unsigned int *__restrict__ keys, int M, int *__restrict__ start,
                                 int *__restrict__ end)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const unsigned int k = keys[i];
  if (k == 0) return;                                     // no word
  if (i == 0 || keys[i - 1] != k) start[k - 1] = i;
  if (i == M - 1 || keys[i + 1] != k) end[k - 1] = i + 1;
}

// One CTA per word: thread c sums component c over the members in ascending global id (float64, from 0); thread 0
// sums the 128 squares in ascending c; the word becomes float32(s_c / sqrt(norm)).  A word without members (or with a
// zero sum) keeps its descriptor.
__global__ void __launch_bounds__(128)
vb_update_kernel(const VbSet *__restrict__ sets, int numSets, const int *__restrict__ sorted,
                 const int *__restrict__ start, const int *__restrict__ end, SiftPoint *__restrict__ vocab,
                 unsigned int *__restrict__ empty)
{
  __shared__ double s_s[128];
  __shared__ double s_norm;
  const int k = blockIdx.x, c = threadIdx.x;
  const int b = start[k], e = end[k];
  if (b == e) {
    if (c == 0) atomicAdd(empty, 1u);
    return;
  }
  double s = 0.0;
  for (int m = b; m < e; m++) s = __dadd_rn(s, (double)vb_desc(sets, numSets, sorted[m])[c]);
  s_s[c] = s;
  __syncthreads();
  if (c == 0) {
    double n = 0.0;
    for (int j = 0; j < 128; j++) n = __dadd_rn(n, __dmul_rn(s_s[j], s_s[j]));
    s_norm = n;
  }
  __syncthreads();
  const double n = s_norm;
  if (n > 0.0) vocab[k].data[c] = __double2float_rn(__ddiv_rn(s, __dsqrt_rn(n)));
}

// The start words: record k is zero but for the descriptor of feature draws[k].
__global__ void vb_start_kernel(const VbSet *__restrict__ sets, int numSets, const int *__restrict__ draws,
                                SiftPoint *__restrict__ vocab)
{
  const int k = blockIdx.x, t = threadIdx.x;             // 144 floats per record, the descriptor from float 16 on
  float v = 0.0f;
  if (t >= 16) v = vb_desc(sets, numSets, draws[k])[t - 16];
  reinterpret_cast<float *>(vocab + k)[t] = v;
}
static_assert(offsetof(SiftPoint, data) == 64 && sizeof(SiftPoint) == 144 * 4, "record layout of vb_start_kernel");

}  // namespace

// The start indices: the k-th distinct idx = ((vp_splitmix64(seed + GOLDEN * counter) >> 32) * M) >> 32 over counter = 0,
// 1, 2, ... (uint64 arithmetic).
std::vector<int> vocab_start_draws(unsigned long long seed, int M, int numWords)
{
  std::vector<int> draws;
  std::vector<unsigned char> seen((size_t)M, 0);
  for (unsigned long long ctr = 0; (int)draws.size() < numWords; ctr++) {
    const unsigned long long x = vp_splitmix64(seed + GOLDEN * ctr);
    const int idx = (int)(((x >> 32) * (unsigned long long)M) >> 32);
    if (!seen[idx]) { seen[idx] = 1; draws.push_back(idx); }
  }
  return draws;
}

int vocab_train(DeviceCtx &c, const cs_match_set *sets, int numSets, int numWords, int maxIterations,
                unsigned long long seed, SiftPoint *vocab, double *trace, long long stats[4])
{
  const cudaStream_t st = c.stream;
  const unsigned long long launches0 = g_launches;
  std::vector<VbSet> hs;
  long long Mll = 0;
  for (int a = 0; a < numSets; a++)
    if (sets[a].n > 0) { hs.push_back(VbSet{static_cast<const SiftPoint *>(sets[a].pts), (int)Mll}); Mll += sets[a].n; }
  const int M = (int)Mll, S = (int)hs.size();
  const std::vector<int> draws = vocab_start_draws(seed, M, numWords);
  const int tiles = idivup(M, VB_TILE);
  const int bits = key_bits((unsigned long long)numWords);
  size_t sortBytes = 0;
  {
    cub::DoubleBuffer<unsigned int> k(nullptr, nullptr);
    cub::DoubleBuffer<int> v(nullptr, nullptr);
    CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sortBytes, k, v, M, 0, bits, st));
  }
  Layout L(256);
  const size_t oSets = L.take(S * sizeof(VbSet)), oDraws = L.take(numWords * sizeof(int));
  const size_t oCur = L.take((size_t)M * 4), oPrev = L.take((size_t)M * 4), oBest = L.take((size_t)M * 4);
  const size_t oK0 = L.take((size_t)M * 4), oK1 = L.take((size_t)M * 4), oV0 = L.take((size_t)M * 4),
               oV1 = L.take((size_t)M * 4);
  const size_t oStart = L.take(numWords * sizeof(int)), oEnd = L.take(numWords * sizeof(int));
  const size_t oPart = L.take(tiles * sizeof(VbPartial)), oEmpty = L.take(sizeof(unsigned int));
  const size_t oTemp = L.take(sortBytes);
  Layout H(256);
  const size_t hSets = H.take(S * sizeof(VbSet)), hDraws = H.take(numWords * sizeof(int));
  const size_t hPart = H.take(tiles * sizeof(VbPartial)), hEmpty = H.take((maxIterations + 1) * sizeof(unsigned int));
  int r;
  if ((r = c.vocab.grow(L.bytes)) < 0 || (r = c.h_vocab.grow(H.bytes)) < 0) return r;
  char *d = c.vocab.as<char>(), *h = c.h_vocab.as<char>();
  VbSet *dSets = reinterpret_cast<VbSet *>(d + oSets);
  int *dDraws = reinterpret_cast<int *>(d + oDraws), *cur = reinterpret_cast<int *>(d + oCur);
  int *prev = reinterpret_cast<int *>(d + oPrev);
  float *best = reinterpret_cast<float *>(d + oBest);
  unsigned int *k0 = reinterpret_cast<unsigned int *>(d + oK0), *k1 = reinterpret_cast<unsigned int *>(d + oK1);
  int *v0 = reinterpret_cast<int *>(d + oV0), *v1 = reinterpret_cast<int *>(d + oV1);
  int *start = reinterpret_cast<int *>(d + oStart), *end = reinterpret_cast<int *>(d + oEnd);
  VbPartial *part = reinterpret_cast<VbPartial *>(d + oPart);
  unsigned int *empty = reinterpret_cast<unsigned int *>(d + oEmpty);
  const VbPartial *hp = reinterpret_cast<const VbPartial *>(h + hPart);
  unsigned int *he = reinterpret_cast<unsigned int *>(h + hEmpty);
  std::copy(hs.begin(), hs.end(), reinterpret_cast<VbSet *>(h + hSets));
  std::copy(draws.begin(), draws.end(), reinterpret_cast<int *>(h + hDraws));
  CS_CUDA(cudaMemcpyAsync(d + oSets, h + hSets, hDraws + numWords * sizeof(int), cudaMemcpyHostToDevice, st));
  vb_start_kernel<<<numWords, 144, 0, st>>>(dSets, S, dDraws, vocab);
  count_launch();
  CS_CUDA(cudaGetLastError());
  for (int t = 0; t < 4 * maxIterations; t++) trace[t] = 0.0;
  int iterations = 0, stopped = 0;
  for (int t = 0; t < maxIterations; t++) {
    VocabAssign va;
    if ((r = vocab_assign_enqueue(c, sets, numSets, vocab, numWords, cur, best, va)) < 0) return r;
    vb_compare_kernel<<<tiles, VB_THREADS, 0, st>>>(cur, prev, best, M, t == 0, part, k0, v0);
    count_launch();
    CS_CUDA(cudaGetLastError());
    CS_CUDA(cudaMemcpyAsync(h + hPart, part, tiles * sizeof(VbPartial), cudaMemcpyDeviceToHost, st));
    CS_CUDA(cudaStreamSynchronize(st));
    unsigned long long changed = 0, assigned = 0, ast[5];
    double sum = 0.0;
    for (int b = 0; b < tiles; b++) { changed += hp[b].changed; assigned += hp[b].assigned; sum += hp[b].sum; }
    vocab_assign_stats(va, ast);
    double *row = trace + 4 * t;
    row[0] = (double)changed;
    row[2] = (double)ast[2];
    row[3] = assigned ? sum / (double)assigned : 0.0;
    iterations = t + 1;
    if (changed == 0) {                                    // the assignment of iteration t - 1: its empty words
      stopped = 1;
      he[t] = t > 0 ? he[t - 1] : 0;
      break;
    }
    cub::DoubleBuffer<unsigned int> keys(k0, k1);
    cub::DoubleBuffer<int> vals(v0, v1);
    CS_CUDA(cub::DeviceRadixSort::SortPairs(d + oTemp, sortBytes, keys, vals, M, 0, bits, st));
    CS_CUDA(cudaMemsetAsync(start, 0, 2 * (oEnd - oStart), st));   // start and end
    CS_CUDA(cudaMemsetAsync(empty, 0, sizeof(unsigned int), st));
    vb_bounds_kernel<<<idivup(M, 256), 256, 0, st>>>(keys.Current(), M, start, end);
    vb_update_kernel<<<numWords, 128, 0, st>>>(dSets, S, vals.Current(), start, end, vocab, empty);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
    CS_CUDA(cudaMemcpyAsync(he + t, empty, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
  }
  CS_CUDA(cudaStreamSynchronize(st));
  for (int t = 0; t < iterations; t++) trace[4 * t + 1] = (double)he[t];
  stats[0] = iterations;
  stats[1] = stopped;
  stats[2] = M;
  stats[3] = (long long)(g_launches - launches0);
  return iterations;
}

// ------------------------------------------------------------------------------ retrieval
namespace {

constexpr double RT_Q_SCALE = 4194304.0;          // 2^22
constexpr double RT_SCORE_SCALE = 1.0 / 17592186044416.0;   // 2^-44
constexpr int RT_TOPK_THREADS = 256;
constexpr int RT_TOPK_MAX = 1024;

// A non-empty image and its first global id (table_find on base).
struct RtImage {
  int base, image;
};

// Statistics words (unsigned long long): [0] N', [1] postings, [2] sum df^2, [3] score updates, [4] waves (host),
// [5] pairs, [6] ignored features.
struct RtBufs {
  const int *wordOf;
  int N, numImages, numWords;
  const RtImage *images; int numNonEmpty;
  unsigned long long *keys;       // (image, word) keys, sorted into keys2
  unsigned long long *uniq;       // the runs' keys
  int *tf;                        // the runs' lengths
  int *numRuns;
  int *postImg, *postWord, *postQ;
  unsigned int *wordKey[2]; int *wordVal[2];
  int *df, *dfq, *wBegin, *wEnd, *imgBegin, *imgEnd;
  double *idf;
  unsigned long long *stats;
};

__global__ void rt_keys_kernel(RtBufs b)
{
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= b.N) return;
  const unsigned long long sentinel = (unsigned long long)b.numImages * b.numWords;
  const int w = b.wordOf[g];
  unsigned long long key = sentinel;
  if (w >= 0 && w < b.numWords) {
    const int a = b.images[table_find(b.images, b.numNonEmpty, &RtImage::base, g)].image;
    key = (unsigned long long)a * b.numWords + w;
  } else {
    atomicAdd(&b.stats[6], 1ull);
  }
  b.keys[g] = key;
}

// Per run p (a posting, or the sentinel run of the ignored features): image, word, df, the image bounds, N'.  Every
// p < N also clears its word-sort key.
__global__ void rt_postings_kernel(RtBufs b)
{
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= b.N) return;
  b.wordKey[0][p] = (unsigned int)b.numWords;
  b.wordVal[0][p] = p;
  if (p >= *b.numRuns) return;
  const unsigned long long sentinel = (unsigned long long)b.numImages * b.numWords;
  const unsigned long long key = b.uniq[p];
  if (key == sentinel) return;
  const int a = (int)(key / b.numWords), w = (int)(key % b.numWords);
  b.postImg[p] = a;
  b.postWord[p] = w;
  atomicAdd(&b.df[w], 1);
  atomicAdd(&b.stats[1], 1ull);
  if (p == 0 || (int)(b.uniq[p - 1] / b.numWords) != a) { b.imgBegin[a] = p; atomicAdd(&b.stats[0], 1ull); }
  if (p + 1 == *b.numRuns || b.uniq[p + 1] == sentinel || (int)(b.uniq[p + 1] / b.numWords) != a) b.imgEnd[a] = p + 1;
}

// idf_w = log(N' / df_w) in float64 (0 for df_w = 0), and sum df_w^2.
__global__ void rt_idf_kernel(RtBufs b, double *__restrict__ out)
{
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= b.numWords) return;
  const int d = b.df[w];
  const double v = d > 0 ? log((double)b.stats[0] / (double)d) : 0.0;
  b.idf[w] = v;
  if (out) out[w] = v;
  if (d > 0) atomicAdd(&b.stats[2], (unsigned long long)d * (unsigned long long)d);
}

// One warp per image: lane 0 sums (tf idf)^2 over its postings in ascending word (float64, from 0, no contraction),
// then every lane q = rint(tf idf / sqrt(norm) * 2^22) for its postings (0 when the norm is 0).  Postings with q != 0
// get their word as sort key (the others keep numWords: not in the inverted file).
__global__ void rt_weights_kernel(RtBufs b)
{
  const int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (a >= b.numImages) return;
  const int p0 = b.imgBegin[a], p1 = b.imgEnd[a];
  double norm = 0.0;
  if (lane == 0)
    for (int p = p0; p < p1; p++) {
      const double x = __dmul_rn((double)b.tf[p], b.idf[b.postWord[p]]);
      norm = __dadd_rn(norm, __dmul_rn(x, x));
    }
  norm = __shfl_sync(0xffffffffu, norm, 0);
  const double s = __dsqrt_rn(norm);
  for (int p = p0 + lane; p < p1; p += 32) {
    const int w = b.postWord[p];
    const double x = __dmul_rn((double)b.tf[p], b.idf[w]);
    const int q = norm > 0.0 ? __double2int_rn(__dmul_rn(__ddiv_rn(x, s), RT_Q_SCALE)) : 0;
    b.postQ[p] = q;
    if (q != 0) {
      b.wordKey[0][p] = (unsigned int)w;
      atomicAdd(&b.dfq[w], 1);
    }
  }
}

// The inverted file's word bounds, and sum dfq_w^2 (the score updates).
__global__ void rt_bounds_kernel(RtBufs b, const unsigned int *__restrict__ keys)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < b.numWords) {
    const unsigned long long d = (unsigned long long)b.dfq[i];
    if (d) atomicAdd(&b.stats[3], d * d);
  }
  if (i >= b.N) return;
  const unsigned int k = keys[i];
  if (k >= (unsigned int)b.numWords) return;
  if (i == 0 || keys[i - 1] != k) b.wBegin[k] = i;
  if (i == b.N - 1 || keys[i + 1] != k) b.wEnd[k] = i + 1;
}

__device__ __forceinline__ int rt_lower_bound(const int *__restrict__ a, int n, int x)
{
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// The queries [a0, a1): one warp per posting of a query (postings are in image order), its lanes over the inverted
// list of the posting's word; acc[a - a0][b] += q_a q_b (exact uint64 atomics).
__global__ void __launch_bounds__(256)
rt_scatter_kernel(RtBufs b, const int *__restrict__ inv, int a0, int a1, unsigned long long *__restrict__ acc)
{
  const int P = (int)b.stats[1];
  const int p0 = rt_lower_bound(b.postImg, P, a0), p1 = rt_lower_bound(b.postImg, P, a1);
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < p1 - p0; p += warps) {
    const int pp = p0 + p, q = b.postQ[pp];
    if (q == 0) continue;
    const int w = b.postWord[pp];
    unsigned long long *row = acc + (size_t)(b.postImg[pp] - a0) * b.numImages;
    for (int i = b.wBegin[w] + lane; i < b.wEnd[w]; i += 32) {
      const int o = inv[i];
      atomicAdd(&row[b.postImg[o]], (unsigned long long)q * (unsigned long long)b.postQ[o]);
    }
  }
}

// One CTA per query a: the keys (score << 16) | (0xFFFF - b) of the b != a with score > 0, the topK largest by a
// radix select (8-bit digits from bit 56; keys are unique), sorted descending (bitonic, in shared memory).  Writes the
// neighbours, the similarities score * 2^-44 and the candidate pair keys min(a, b) << 16 | max(a, b) (0xFFFFFFFF:
// none).
__global__ void __launch_bounds__(RT_TOPK_THREADS)
rt_topk_kernel(const unsigned long long *__restrict__ acc, int numImages, int a0, int topK, int *__restrict__ nb,
               double *__restrict__ sc, unsigned int *__restrict__ cand)
{
  __shared__ unsigned int hist[256];
  __shared__ unsigned long long s_keys[RT_TOPK_MAX];
  __shared__ unsigned long long s_prefix, s_mask;
  __shared__ int s_need, s_n;
  const int t = threadIdx.x, a = a0 + blockIdx.x;
  const unsigned long long *row = acc + (size_t)blockIdx.x * numImages;
  auto key = [&](int bb) -> unsigned long long {
    const unsigned long long s = row[bb];
    return (bb == a || s == 0) ? 0ull : (s << 16) | (unsigned long long)(0xFFFF - bb);
  };
  if (t == 0) { s_prefix = 0; s_mask = 0; s_n = 0; }
  __syncthreads();
  // the number of positive keys
  int cnt = 0;
  for (int bb = t; bb < numImages; bb += RT_TOPK_THREADS) cnt += key(bb) != 0;
  atomicAdd(&s_n, cnt);
  __syncthreads();
  cnt = s_n;
  __syncthreads();
  if (t == 0) s_n = 0;
  __syncthreads();
  const int K = cnt < topK ? cnt : topK;
  unsigned long long thresh = 1;                         // every positive key
  if (cnt > topK) {
    if (t == 0) s_need = topK;
    for (int shift = 56; shift >= 0; shift -= 8) {
      hist[t] = 0;
      __syncthreads();
      const unsigned long long prefix = s_prefix, mask = s_mask;
      for (int bb = t; bb < numImages; bb += RT_TOPK_THREADS) {
        const unsigned long long k = key(bb);
        if (k != 0 && (k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255], 1u);
      }
      __syncthreads();
      if (t == 0) {
        int cum = 0, need = s_need;
        for (int dgt = 255; dgt >= 0; dgt--) {
          if (cum + (int)hist[dgt] >= need) {
            s_need = need - cum;
            s_prefix = prefix | ((unsigned long long)dgt << shift);
            s_mask = mask | (255ull << shift);
            break;
          }
          cum += hist[dgt];
        }
      }
      __syncthreads();
    }
    thresh = s_prefix;
  }
  for (int bb = t; bb < numImages; bb += RT_TOPK_THREADS) {
    const unsigned long long k = key(bb);
    if (k != 0 && k >= thresh) s_keys[atomicAdd(&s_n, 1)] = k;
  }
  int n2 = 1;
  while (n2 < K) n2 <<= 1;
  __syncthreads();
  for (int i = K + t; i < n2; i += RT_TOPK_THREADS) s_keys[i] = 0;
  __syncthreads();
  for (int k = 2; k <= n2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = t; i < n2; i += RT_TOPK_THREADS) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long x = s_keys[i], y = s_keys[ixj];
          const bool desc = (i & k) == 0;
          if (desc ? x < y : x > y) { s_keys[i] = y; s_keys[ixj] = x; }
        }
      }
      __syncthreads();
    }
  for (int j = t; j < topK; j += RT_TOPK_THREADS) {
    const size_t o = (size_t)a * topK + j;
    if (j < K) {
      const unsigned long long k = s_keys[j];
      const int bb = 0xFFFF - (int)(k & 0xFFFF);
      nb[o] = bb;
      sc[o] = (double)(k >> 16) * RT_SCORE_SCALE;
      cand[o] = ((unsigned int)min(a, bb) << 16) | (unsigned int)max(a, bb);
    } else {
      nb[o] = -1;
      sc[o] = 0.0;
      cand[o] = 0xFFFFFFFFu;
    }
  }
}

// The deduplicated pairs: count = unique keys without the 0xFFFFFFFF key; the first min(count, maxPairs) written.
__global__ void rt_pairs_kernel(const unsigned int *__restrict__ uniq, const int *__restrict__ numUnique,
                                int2 *__restrict__ pairs, int maxPairs, unsigned long long *__restrict__ stats)
{
  const int u = *numUnique;
  const int count = u > 0 && uniq[u - 1] == 0xFFFFFFFFu ? u - 1 : u;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) stats[5] = (unsigned long long)count;
  if (i < count && i < maxPairs) pairs[i] = make_int2((int)(uniq[i] >> 16), (int)(uniq[i] & 0xFFFF));
}

}  // namespace

int retrieve_queries_per_wave(int numImages)
{
  const size_t k = WAVE_BYTES / ((size_t)numImages * sizeof(unsigned long long));
  return k < 1 ? 1 : k > (size_t)numImages ? numImages : (int)k;
}

int retrieve_enqueue(DeviceCtx &c, const int *imageSizes, int numImages, const int *wordOf, int numWords, int topK,
                     int *neighbours, double *scores, double *idfOut, int *pairs, int maxPairs)
{
  const cudaStream_t st = c.stream;
  std::vector<RtImage> imgs;
  long long Nll = 0;
  for (int a = 0; a < numImages; a++)
    if (imageSizes[a] > 0) { imgs.push_back(RtImage{(int)Nll, a}); Nll += imageSizes[a]; }
  const int N = (int)Nll, I = numImages, W = numWords, E = (int)imgs.size();
  const size_t C = (size_t)I * topK;                       // candidate pair keys
  const int perWave = retrieve_queries_per_wave(I), waves = idivup(I, perWave);
  const int keyBits = key_bits((unsigned long long)I * W), wordBits = key_bits((unsigned long long)W);
  // cub's temporary storage: the largest of the five passes
  size_t tmp = 0, x = 0;
  {
    cub::DoubleBuffer<unsigned long long> k64(nullptr, nullptr);
    CS_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, x, k64, N, 0, keyBits, st)); tmp = std::max(tmp, x);
    CS_CUDA(cub::DeviceRunLengthEncode::Encode(nullptr, x, (unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                               (int *)nullptr, (int *)nullptr, N, st));
    tmp = std::max(tmp, x);
    cub::DoubleBuffer<unsigned int> k32(nullptr, nullptr);
    cub::DoubleBuffer<int> v32(nullptr, nullptr);
    CS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, x, k32, v32, N, 0, wordBits, st)); tmp = std::max(tmp, x);
    CS_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, x, k32, (int)C, 0, 32, st)); tmp = std::max(tmp, x);
    CS_CUDA(cub::DeviceSelect::Unique(nullptr, x, (unsigned int *)nullptr, (unsigned int *)nullptr, (int *)nullptr,
                                      (int)C, st));
    tmp = std::max(tmp, x);
  }
  Layout L(256);
  const size_t oStats = L.take(8 * sizeof(unsigned long long)), oImgs = L.take(E * sizeof(RtImage));
  const size_t oK0 = L.take((size_t)N * 8), oK1 = L.take((size_t)N * 8), oUniq = L.take((size_t)N * 8);
  const size_t oTf = L.take((size_t)N * 4), oRuns = L.take(2 * sizeof(int));
  const size_t oPI = L.take((size_t)N * 4), oPW = L.take((size_t)N * 4), oPQ = L.take((size_t)N * 4);
  const size_t oWK0 = L.take((size_t)N * 4), oWK1 = L.take((size_t)N * 4), oWV0 = L.take((size_t)N * 4),
               oWV1 = L.take((size_t)N * 4);
  // cleared together: df, dfq, wBegin, wEnd, imgBegin, imgEnd
  const size_t oDf = L.take((size_t)W * 4), oDfq = L.take((size_t)W * 4), oWB = L.take((size_t)W * 4),
               oWE = L.take((size_t)W * 4), oIB = L.take((size_t)I * 4), oIE = L.take((size_t)I * 4);
  const size_t oIdf = L.take((size_t)W * 8);
  const size_t oAcc = L.take((size_t)perWave * I * 8);
  const size_t oC0 = L.take(C * 4), oC1 = L.take(C * 4), oCU = L.take(C * 4);
  const size_t oTmp = L.take(tmp);
  int r;
  if ((r = c.retrieve.grow(L.bytes)) < 0) return r;
  if ((r = c.h_retrieve.grow(8 * sizeof(unsigned long long) + E * sizeof(RtImage))) < 0) return r;
  char *d = c.retrieve.as<char>();
  char *h = c.h_retrieve.as<char>();
  std::copy(imgs.begin(), imgs.end(), reinterpret_cast<RtImage *>(h + 8 * sizeof(unsigned long long)));
  RtBufs b;
  b.wordOf = wordOf; b.N = N; b.numImages = I; b.numWords = W;
  b.images = reinterpret_cast<const RtImage *>(d + oImgs); b.numNonEmpty = E;
  b.keys = reinterpret_cast<unsigned long long *>(d + oK0);
  b.uniq = reinterpret_cast<unsigned long long *>(d + oUniq);
  b.tf = reinterpret_cast<int *>(d + oTf);
  b.numRuns = reinterpret_cast<int *>(d + oRuns);
  b.postImg = reinterpret_cast<int *>(d + oPI); b.postWord = reinterpret_cast<int *>(d + oPW);
  b.postQ = reinterpret_cast<int *>(d + oPQ);
  b.wordKey[0] = reinterpret_cast<unsigned int *>(d + oWK0); b.wordKey[1] = reinterpret_cast<unsigned int *>(d + oWK1);
  b.wordVal[0] = reinterpret_cast<int *>(d + oWV0); b.wordVal[1] = reinterpret_cast<int *>(d + oWV1);
  b.df = reinterpret_cast<int *>(d + oDf); b.dfq = reinterpret_cast<int *>(d + oDfq);
  b.wBegin = reinterpret_cast<int *>(d + oWB); b.wEnd = reinterpret_cast<int *>(d + oWE);
  b.imgBegin = reinterpret_cast<int *>(d + oIB); b.imgEnd = reinterpret_cast<int *>(d + oIE);
  b.idf = reinterpret_cast<double *>(d + oIdf);
  b.stats = reinterpret_cast<unsigned long long *>(d + oStats);
  void *temp = d + oTmp;
  unsigned long long *acc = reinterpret_cast<unsigned long long *>(d + oAcc);
  unsigned int *cand0 = reinterpret_cast<unsigned int *>(d + oC0), *cand1 = reinterpret_cast<unsigned int *>(d + oC1);
  unsigned int *candU = reinterpret_cast<unsigned int *>(d + oCU);

  CS_CUDA(cudaMemsetAsync(d + oStats, 0, 8 * sizeof(unsigned long long), st));
  CS_CUDA(cudaMemsetAsync(d + oDf, 0, oIdf - oDf, st));
  if (E) CS_CUDA(cudaMemcpyAsync(d + oImgs, h + 8 * sizeof(unsigned long long), E * sizeof(RtImage),
                                 cudaMemcpyHostToDevice, st));
  const int g256 = idivup(std::max(N, 1), 256);
  rt_keys_kernel<<<g256, 256, 0, st>>>(b);
  cub::DoubleBuffer<unsigned long long> k64(b.keys, reinterpret_cast<unsigned long long *>(d + oK1));
  CS_CUDA(cub::DeviceRadixSort::SortKeys(temp, tmp, k64, N, 0, keyBits, st));
  CS_CUDA(cub::DeviceRunLengthEncode::Encode(temp, tmp, k64.Current(), b.uniq, b.tf, b.numRuns, N, st));
  rt_postings_kernel<<<g256, 256, 0, st>>>(b);
  rt_idf_kernel<<<idivup(W, 256), 256, 0, st>>>(b, idfOut);
  rt_weights_kernel<<<idivup(I, 8), 256, 0, st>>>(b);
  cub::DoubleBuffer<unsigned int> wk(b.wordKey[0], b.wordKey[1]);
  cub::DoubleBuffer<int> wv(b.wordVal[0], b.wordVal[1]);
  CS_CUDA(cub::DeviceRadixSort::SortPairs(temp, tmp, wk, wv, N, 0, wordBits, st));
  rt_bounds_kernel<<<idivup(std::max(N, W), 256), 256, 0, st>>>(b, wk.Current());
  count_launch(5);
  CS_CUDA(cudaGetLastError());
  for (int a0 = 0; a0 < I; a0 += perWave) {
    const int a1 = std::min(I, a0 + perWave);
    CS_CUDA(cudaMemsetAsync(acc, 0, (size_t)(a1 - a0) * I * 8, st));
    rt_scatter_kernel<<<8 * c.sms, 256, 0, st>>>(b, wv.Current(), a0, a1, acc);
    rt_topk_kernel<<<a1 - a0, RT_TOPK_THREADS, 0, st>>>(acc, I, a0, topK, neighbours, scores, cand0);
    count_launch(2);
    CS_CUDA(cudaGetLastError());
  }
  cub::DoubleBuffer<unsigned int> ck(cand0, cand1);
  CS_CUDA(cub::DeviceRadixSort::SortKeys(temp, tmp, ck, (int)C, 0, 32, st));
  CS_CUDA(cub::DeviceSelect::Unique(temp, tmp, ck.Current(), candU, b.numRuns + 1, (int)C, st));
  const int room = (int)std::min<size_t>(C, (size_t)maxPairs);
  rt_pairs_kernel<<<idivup(std::max(room, 1), 256), 256, 0, st>>>(candU, b.numRuns + 1,
                                                                  reinterpret_cast<int2 *>(pairs), maxPairs, b.stats);
  count_launch();
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaMemcpyAsync(h, b.stats, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  c.retrieveWaves = waves;
  return 0;
}

}  // namespace cs
