// match_mutual.cu -- the pair lists of a mutual match and of a ratio match, built as the ordered lists of
// ordered_list.cuh (flag, then scan and write; no atomics, so the order follows from the values).
// Mutual: the pairs (i, j) with
//   s1[i].match == j >= 0,  s2[j].match == i,  s1[i].score > minScore,  s1[i].ambiguity < maxAmbiguity
// (strict comparisons, as FindHomography, homography.cu:200), written as int2 {i, j} in increasing i.  Every j
// appears at most once (it pairs only with i = s2[j].match).  Two launches: mutual_flags_kernel, then
// mutual_write_kernel, which writes the pairs at positions < maxPairs and the total.
// Ratio (cs_match_ratio): the same two launches on the two-nearest-neighbour lists; ratio_flags_kernel applies Lowe's
// ratio test (COLMAP's rule, on angles) and the optional cross-check, and the write kernel reads j = idx[i][0].
#include "common.cuh"
#include "ordered_list.cuh"

namespace cs {

__global__ void __launch_bounds__(LIST_ROWS)
mutual_flags_kernel(const SiftPoint *__restrict__ s1, int n1, const SiftPoint *__restrict__ s2, int n2, float minScore,
                    float maxAmbiguity, unsigned int *__restrict__ masks, unsigned int *__restrict__ blockCounts)
{
  const int i = blockIdx.x * LIST_ROWS + threadIdx.x;
  bool keep = false;
  if (i < n1) {
    const int j = s1[i].match;
    if (j >= 0 && j < n2 && s1[i].score > minScore && s1[i].ambiguity < maxAmbiguity) keep = __ldg(&s2[j].match) == i;
  }
  list_flag(keep, i, n1, masks, blockCounts, blockIdx.x);
}

// The pair list of this CTA and the CTA's index in it: the one of a call, or job k of a batch table (jobs != nullptr).
__device__ __forceinline__ PairJob pair_job(const PairJob &one, const PairJob *__restrict__ jobs, int numJobs, int &blk)
{
  if (!jobs) { blk = blockIdx.x; return one; }
  const PairJob j = jobs[table_find(jobs, numJobs, &PairJob::cta0, (int)blockIdx.x)];
  blk = (int)blockIdx.x - j.cta0;
  return j;
}

// The pairs {i, jv[i * jstride]} of the kept rows at their positions within the CTA's pair list, and the total.
__global__ void __launch_bounds__(LIST_ROWS)
mutual_write_kernel(const PairJob one, const PairJob *__restrict__ jobs, int numJobs)
{
  int blk;
  const PairJob pj = pair_job(one, jobs, numJobs, blk);
  bool bit;
  const unsigned int pos = list_position(pj.masks, pj.blockCounts, pj.n1, blk, &bit, pj.total);
  const int i = blk * LIST_ROWS + threadIdx.x;
  if (bit && pos < (unsigned int)pj.maxPairs) pj.pairs[pos] = make_int2(i, pj.jv[(size_t)i * pj.jstride]);
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
__global__ void __launch_bounds__(LIST_ROWS)
ratio_flags_kernel(const PairJob one, const PairJob *__restrict__ jobs, int numJobs, double maxRatio, double maxDistance)
{
  int blk;
  const PairJob pj = pair_job(one, jobs, numJobs, blk);
  const int2 *__restrict__ idx1 = pj.idx1, *__restrict__ idx2 = pj.idx2;
  const float2 *__restrict__ score1 = pj.score1, *__restrict__ score2 = pj.score2;
  const int n1 = pj.n1, n2 = pj.n2;
  const int i = blk * LIST_ROWS + threadIdx.x;
  bool keep = false;
  if (i < n1 && ratio_keep(idx1, score1, i, maxRatio, maxDistance)) {
    keep = true;
    if (idx2) {
      const int j = idx1[i].x;
      keep = j < n2 && idx2[j].x == i && ratio_keep(idx2, score2, j, maxRatio, maxDistance);
    }
  }
  list_flag(keep, i, n1, pj.masks, pj.blockCounts, blk);
}

// Ballot words, CTA counts and the total of n1 rows in c.pairScratch; the total is copied to *c.h_pairTotal after the
// two launches.
static int pairs_scratch(DeviceCtx &c, int n1, PairJob &pj)
{
  const int blocks = list_ctas(n1), words = list_words(n1);
  int r;
  if ((r = c.pairScratch.grow(((size_t)words + blocks + 1) * sizeof(unsigned int))) < 0) return r;
  pj.n1 = n1;
  pj.masks = c.pairScratch.as<unsigned int>(); pj.blockCounts = pj.masks + words; pj.total = pj.blockCounts + blocks;
  pj.cta0 = 0;
  return 0;
}

int launch_mutual_pairs(DeviceCtx &c, const SiftPoint *s1, int n1, const SiftPoint *s2, int n2, const MutualArgs &mu)
{
  PairJob pj = {};
  int r;
  if ((r = pairs_scratch(c, n1, pj)) < 0) return r;
  pj.jv = &s1[0].match; pj.jstride = (int)(sizeof(SiftPoint) / sizeof(int));
  pj.pairs = mu.pairs; pj.maxPairs = mu.maxPairs;
  const int blocks = list_ctas(n1);
  mutual_flags_kernel<<<blocks, LIST_ROWS, 0, c.stream>>>(s1, n1, s2, n2, mu.minScore, mu.maxAmbiguity, pj.masks,
                                                          pj.blockCounts);
  mutual_write_kernel<<<blocks, LIST_ROWS, 0, c.stream>>>(pj, nullptr, 0);
  count_launch(2);
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaMemcpyAsync(c.h_pairTotal, pj.total, sizeof(unsigned int), cudaMemcpyDeviceToHost, c.stream));
  return 0;
}

int launch_ratio_pairs(DeviceCtx &c, const int *idx1, const float *score1, int n1, const int *idx2, const float *score2,
                       int n2, const RatioArgs &ra)
{
  PairJob pj = {};
  int r;
  if ((r = pairs_scratch(c, n1, pj)) < 0) return r;
  pj.jv = idx1; pj.jstride = 2; pj.n2 = n2;
  pj.idx1 = reinterpret_cast<const int2 *>(idx1); pj.score1 = reinterpret_cast<const float2 *>(score1);
  pj.idx2 = reinterpret_cast<const int2 *>(idx2); pj.score2 = reinterpret_cast<const float2 *>(score2);
  pj.pairs = ra.pairs; pj.maxPairs = ra.maxPairs;
  const int blocks = list_ctas(n1);
  ratio_flags_kernel<<<blocks, LIST_ROWS, 0, c.stream>>>(pj, nullptr, 0, (double)ra.maxRatio, (double)ra.maxDistance);
  mutual_write_kernel<<<blocks, LIST_ROWS, 0, c.stream>>>(pj, nullptr, 0);
  count_launch(2);
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaMemcpyAsync(c.h_pairTotal, pj.total, sizeof(unsigned int), cudaMemcpyDeviceToHost, c.stream));
  return 0;
}

// A batch wave: the ratio test and the pair writes of every job of the table, each job's CTAs from its cta0 on.
int launch_ratio_pairs_batch(DeviceCtx &c, const PairJob *jobs, int numJobs, int numCtas, float maxRatio,
                             float maxDistance)
{
  const PairJob none = {};
  ratio_flags_kernel<<<numCtas, LIST_ROWS, 0, c.stream>>>(none, jobs, numJobs, (double)maxRatio, (double)maxDistance);
  mutual_write_kernel<<<numCtas, LIST_ROWS, 0, c.stream>>>(none, jobs, numJobs);
  count_launch(2);
  CS_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace cs
