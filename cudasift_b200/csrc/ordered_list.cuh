// ordered_list.cuh -- the keep-bit lists written on the device without atomics, so that their order follows from the
// values alone: mutual pairs and ratio-test pairs (single, batched and guided; match_mutual.cu), verification's
// valid pairs and its inliers (verify.cu) and fused points (stereo.cu).  Each is built in three steps:
//   1. flag    one thread per row computes a keep bit; one ballot word per 32 rows and one count per CTA of LIST_ROWS
//              rows (list_flag);
//   2. scan    every CTA sums the counts of the CTAs before it, then scans its own ballot words (list_position);
//   3. write   every kept row writes its entry at its exclusive position; the CTA that holds the last row writes the
//              total.
// The scratch of an n-row list is list_words(n) ballot words and list_ctas(n) CTA counts (match_tc.cu and
// match_guided.cu size their waves' pair scratch by them).  Lists where a thread emits any number of entries are the
// counted lists of counted_list.cuh.
#pragma once

namespace cs {

constexpr int LIST_ROWS = 1024;      // rows per CTA of every flag, compact and write kernel (one per thread)

__host__ __device__ inline int list_words(int n) { return (n + 31) / 32; }
__host__ __device__ inline int list_ctas(int n) { return (n + LIST_ROWS - 1) / LIST_ROWS; }

// Step 1 in CTA blk of an n-row list, row = blk * LIST_ROWS + threadIdx.x: the CTA's ballot words and its count.
__device__ __forceinline__ void list_flag(bool keep, int row, int n, unsigned int *__restrict__ masks,
                                          unsigned int *__restrict__ counts, int blk)
{
  const unsigned int bal = __ballot_sync(0xffffffffu, keep);
  if ((threadIdx.x & 31) == 0 && row < n) masks[row >> 5] = bal;
  const int cnt = __syncthreads_count(keep);
  if (threadIdx.x == 0) counts[blk] = (unsigned int)cnt;
}

// Step 2 in CTA blk of an n-row list: this thread's exclusive position among the kept rows, and its own keep bit in
// *bit.  The CTA that holds row n - 1 writes the total to *total when total is given.  Every thread of the CTA calls it.
__device__ __forceinline__ unsigned int list_position(const unsigned int *__restrict__ masks,
                                                      const unsigned int *__restrict__ counts, int n, int blk, bool *bit,
                                                      unsigned int *total)
{
  __shared__ unsigned int s_w[32];
  __shared__ unsigned int s_base;
  const unsigned int FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  // exclusive prefix of this CTA: the counts of the CTAs before it, one per thread for lists of up to LIST_ROWS^2 rows
  // (a deeper unroll only costs registers)
  unsigned int part = 0;
#pragma unroll 4
  for (int k = threadIdx.x; k < blk; k += LIST_ROWS) part += counts[k];
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
  const unsigned int bal = (blk * LIST_ROWS + w * 32 < n) ? masks[(blk * LIST_ROWS >> 5) + w] : 0u;
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
    if (total && lane == 31 && blk == (n - 1) / LIST_ROWS) *total = base + inc;
  }
  __syncthreads();
  *bit = (bal >> lane) & 1u;
  return base + s_w[w] + __popc(bal & ((1u << lane) - 1u));
}

}  // namespace cs
