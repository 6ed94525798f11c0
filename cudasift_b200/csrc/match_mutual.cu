// match_mutual.cu -- the pair lists of a mutual match and of a ratio match.
// Mutual: the pairs (i, j) with
//   s1[i].match == j >= 0,  s2[j].match == i,  s1[i].score > minScore,  s1[i].ambiguity < maxAmbiguity
// (strict comparisons, as FindHomography, homography.cu:200), written as int2 {i, j} in increasing i.  Every j
// appears at most once (it pairs only with i = s2[j].match).  The order is defined by value: two launches, no atomics.
//   1. flags   one thread per row i: the keep test; a ballot word per 32 rows and a count per CTA of 1024 rows.
//   2. write   every CTA sums the counts of the CTAs before it (its exclusive prefix), scans its own 32 ballot words
//              and writes its pairs; the last CTA writes the total.  Pairs at positions >= maxPairs are not written.
// Ratio (cs_match_ratio): the same two launches on the two-nearest-neighbour lists; ratio_flags_kernel applies Lowe's
// ratio test (COLMAP's rule, on angles) and the optional cross-check, and the write kernel reads j = idx[i][0].
#include "common.cuh"

namespace cs {

#define MP_ROWS 1024          // rows per CTA (one per thread)

__global__ void __launch_bounds__(MP_ROWS)
mutual_flags_kernel(const SiftPoint *__restrict__ s1, int n1, const SiftPoint *__restrict__ s2, int n2, float minScore,
                    float maxAmbiguity, unsigned int *__restrict__ masks, unsigned int *__restrict__ blockCounts)
{
  const int i = blockIdx.x * MP_ROWS + threadIdx.x;
  bool keep = false;
  if (i < n1) {
    const int j = s1[i].match;
    if (j >= 0 && j < n2 && s1[i].score > minScore && s1[i].ambiguity < maxAmbiguity) keep = __ldg(&s2[j].match) == i;
  }
  const unsigned int bal = __ballot_sync(0xffffffffu, keep);
  if ((threadIdx.x & 31) == 0 && i < n1) masks[i >> 5] = bal;
  const int cnt = __syncthreads_count(keep);
  if (threadIdx.x == 0) blockCounts[blockIdx.x] = (unsigned int)cnt;
}

__global__ void __launch_bounds__(MP_ROWS)
mutual_write_kernel(const int *__restrict__ jv, int jstride, int n1, const unsigned int *__restrict__ masks,
                    const unsigned int *__restrict__ blockCounts, int2 *__restrict__ pairs, int maxPairs,
                    unsigned int *__restrict__ total)
{
  __shared__ unsigned int s_w[32];
  __shared__ unsigned int s_base;
  const unsigned int FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  // exclusive prefix of this CTA: the counts of the CTAs before it
  unsigned int part = 0;
  for (int k = threadIdx.x; k < (int)blockIdx.x; k += MP_ROWS) part += blockCounts[k];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(FULL, part, o);
  if (lane == 0) s_w[w] = part;
  __syncthreads();
  if (w == 0) {
    unsigned int v = s_w[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    if (lane == 0) s_base = v;
  }
  __syncthreads();
  const unsigned int base = s_base;
  // positions inside the CTA: exclusive scan of the warps' ballot counts
  const int i = blockIdx.x * MP_ROWS + threadIdx.x;
  const unsigned int bal = (blockIdx.x * MP_ROWS + w * 32 < n1) ? masks[(blockIdx.x * MP_ROWS >> 5) + w] : 0u;
  if (lane == 0) s_w[w] = __popc(bal);
  __syncthreads();
  if (w == 0) {
    const unsigned int c = s_w[lane];
    unsigned int inc = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int t = __shfl_up_sync(FULL, inc, o);
      if (lane >= o) inc += t;
    }
    s_w[lane] = inc - c;
    if (lane == 31 && blockIdx.x == gridDim.x - 1) *total = base + inc;
  }
  __syncthreads();
  if ((bal >> lane) & 1u) {
    const unsigned int pos = base + s_w[w] + __popc(bal & ((1u << lane) - 1u));
    if (pos < (unsigned int)maxPairs) pairs[pos] = make_int2(i, jv[(size_t)i * jstride]);
  }
}

// COLMAP's one-way test on row i's two neighbours, in double: d = acos(min(score, 1)), keep when j1 >= 0,
// d1 <= maxDistance and d1 < maxRatio * d2 (a missing second neighbour has score 0, d2 = pi / 2).
__device__ __forceinline__ bool ratio_keep(const int2 *__restrict__ idx, const float2 *__restrict__ score, int i,
                                           double maxRatio, double maxDistance)
{
  const int2 j = idx[i];
  if (j.x < 0) return false;
  const float2 s = score[i];
  const double d1 = acos(fmin((double)s.x, 1.0)), d2 = acos(fmin((double)s.y, 1.0));
  return d1 <= maxDistance && d1 < maxRatio * d2;
}

// one thread per row i of set 1; idx2 != nullptr: cross-check, row j1 of set 2 must pass as well and name i
__global__ void __launch_bounds__(MP_ROWS)
ratio_flags_kernel(const int2 *__restrict__ idx1, const float2 *__restrict__ score1, int n1, const int2 *__restrict__ idx2,
                   const float2 *__restrict__ score2, int n2, double maxRatio, double maxDistance,
                   unsigned int *__restrict__ masks, unsigned int *__restrict__ blockCounts)
{
  const int i = blockIdx.x * MP_ROWS + threadIdx.x;
  bool keep = false;
  if (i < n1 && ratio_keep(idx1, score1, i, maxRatio, maxDistance)) {
    keep = true;
    if (idx2) {
      const int j = idx1[i].x;
      keep = j < n2 && idx2[j].x == i && ratio_keep(idx2, score2, j, maxRatio, maxDistance);
    }
  }
  const unsigned int bal = __ballot_sync(0xffffffffu, keep);
  if ((threadIdx.x & 31) == 0 && i < n1) masks[i >> 5] = bal;
  const int cnt = __syncthreads_count(keep);
  if (threadIdx.x == 0) blockCounts[blockIdx.x] = (unsigned int)cnt;
}

// Ballot words, CTA counts and the total of n1 rows in c.pairScratch; the total is copied to *c.h_pairTotal after the
// two launches.
static int pairs_scratch(DeviceCtx &c, int n1, unsigned int **masks, unsigned int **counts, unsigned int **total)
{
  const int blocks = idivup(n1, MP_ROWS), words = idivup(n1, 32);
  int r;
  if ((r = c.pairScratch.grow(((size_t)words + blocks + 1) * sizeof(unsigned int))) < 0) return r;
  if (!c.h_pairTotal) CS_CUDA(cudaMallocHost((void **)&c.h_pairTotal, sizeof(unsigned int)));
  *masks = c.pairScratch.as<unsigned int>(); *counts = *masks + words; *total = *counts + blocks;
  return 0;
}

int launch_mutual_pairs(DeviceCtx &c, const SiftPoint *s1, int n1, const SiftPoint *s2, int n2, const MutualArgs &mu)
{
  unsigned int *masks, *counts, *total;
  int r;
  if ((r = pairs_scratch(c, n1, &masks, &counts, &total)) < 0) return r;
  const int blocks = idivup(n1, MP_ROWS);
  mutual_flags_kernel<<<blocks, MP_ROWS, 0, c.stream>>>(s1, n1, s2, n2, mu.minScore, mu.maxAmbiguity, masks, counts);
  mutual_write_kernel<<<blocks, MP_ROWS, 0, c.stream>>>(&s1[0].match, (int)(sizeof(SiftPoint) / sizeof(int)), n1, masks,
                                                        counts, mu.pairs, mu.maxPairs, total);
  count_launch(2);
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaMemcpyAsync(c.h_pairTotal, total, sizeof(unsigned int), cudaMemcpyDeviceToHost, c.stream));
  return 0;
}

int launch_ratio_pairs(DeviceCtx &c, const int *idx1, const float *score1, int n1, const int *idx2, const float *score2,
                       int n2, const RatioArgs &ra)
{
  unsigned int *masks, *counts, *total;
  int r;
  if ((r = pairs_scratch(c, n1, &masks, &counts, &total)) < 0) return r;
  const int blocks = idivup(n1, MP_ROWS);
  ratio_flags_kernel<<<blocks, MP_ROWS, 0, c.stream>>>(reinterpret_cast<const int2 *>(idx1),
                                                       reinterpret_cast<const float2 *>(score1), n1,
                                                       reinterpret_cast<const int2 *>(idx2),
                                                       reinterpret_cast<const float2 *>(score2), n2, (double)ra.maxRatio,
                                                       (double)ra.maxDistance, masks, counts);
  mutual_write_kernel<<<blocks, MP_ROWS, 0, c.stream>>>(idx1, 2, n1, masks, counts, ra.pairs, ra.maxPairs, total);
  count_launch(2);
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaMemcpyAsync(c.h_pairTotal, total, sizeof(unsigned int), cudaMemcpyDeviceToHost, c.stream));
  return 0;
}

}  // namespace cs
