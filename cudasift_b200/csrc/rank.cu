// rank.cu -- ranked extraction: per image, the maxOut records with the largest |sharpness|, in a fixed order.
//
// Rank key, first field first: |sharpness| descending, then subsampling, ypos, xpos, scale, orientation ascending
// (numpy: lexsort((orientation, scale, xpos, ypos, subsampling, -abs(sharpness)))).  A keypoint's secondary orientation
// equals its primary on the first five fields, so the sixth orders the pair.  The result depends on the values of
// the candidate records only, never on the order in which the detector's atomics placed them.
//
// Three launches per batch, all reading the counts on the device:
//   rank_select_kernel  one CTA per image: radix select (8-bit digits) of the keep-th |sharpness| key, then
//                       compaction of every candidate at or above it (ties at the threshold included) with its full key
//   rank_order_kernel   a 2-D grid of CTAs per image (survivor tiles x survivor tiles): rank of each survivor = number
//                       of survivors with a smaller full key, summed over the tiles with one atomic per survivor and
//                       tile; ranks below keep are the output positions
//   rank_gather_kernel  one warp per survivor of rank < keep: 36 uint4 copies from the candidate area to the slot
#include "common.cuh"

namespace cs {

#define RK_SELECT_THREADS 1024
#define RK_ORDER_THREADS 256
#define RK_GATHER_THREADS 256
#define RK_KEY_WORDS 6        // |sharpness| (descending), subsampling, ypos, xpos, scale, orientation

static_assert(RK_KEY_WORDS + 3 == CS_RANK_SCRATCH_PER_IN, "scratch layout (common.cuh)");

struct RankImage {
  const SiftPoint *in;
  SiftPoint *out;
  unsigned int *cnt, *keys, *sk, *rank, *nsurv;
};

__device__ __forceinline__ RankImage rank_image(const RankParams &P, int img)
{
  RankImage r;
  r.in = P.in + (size_t)img * P.inStride;
  r.out = P.out + (size_t)img * P.outStride;
  r.cnt = P.counters + (size_t)img * CS_CNT_STRIDE;
  r.keys = P.scratch + (size_t)img * rank_scratch_words(P.maxIn);
  r.sk = r.keys + P.maxIn;
  r.rank = r.sk + (size_t)(RK_KEY_WORDS + 1) * P.maxIn;
  r.nsurv = r.rank + P.maxIn;
  return r;
}

// |sharpness| descending as an ascending unsigned key (fabsf clears the sign, so -0 and +0 agree)
__device__ __forceinline__ unsigned int rank_key0(float sharpness) { return ~__float_as_uint(fabsf(sharpness)); }

// IEEE order as unsigned order; -0 is mapped to +0 because the two compare equal
__device__ __forceinline__ unsigned int ord_key(float v)
{
  unsigned int u = __float_as_uint(v);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// records in the candidate area: the extractor's count rule (count_from_counters in api.cu)
__device__ __forceinline__ int rank_found(const unsigned int *c, int maxIn)
{
  return (int)max(min(c[0], (unsigned)maxIn), min(c[1], (unsigned)maxIn));
}

__global__ void __launch_bounds__(RK_SELECT_THREADS) rank_select_kernel(const __grid_constant__ RankParams P)
{
  __shared__ unsigned int s_hist[256];
  __shared__ unsigned int s_prefix, s_need, s_count;
  const int tid = threadIdx.x;
  const RankImage I = rank_image(P, blockIdx.x);
  const int n = rank_found(I.cnt, P.maxIn);
  const int keep = min(n, P.maxOut);

  for (int i = tid; i < n; i += RK_SELECT_THREADS) I.keys[i] = rank_key0(I.in[i].sharpness);
  unsigned int thr = 0xffffffffu;                // every candidate survives when all of them are kept
  if (keep < n) {
    // the keep-th smallest key, 8 bits per pass from the top: `need` counts within the keys that share `prefix`
    unsigned int prefix = 0u, need = (unsigned)keep;
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int b = tid; b < 256; b += RK_SELECT_THREADS) s_hist[b] = 0u;
      __syncthreads();
      const unsigned int hmask = shift == 24 ? 0u : (0xffffffffu << (shift + 8));
      for (int i = tid; i < n; i += RK_SELECT_THREADS) {
        const unsigned int k = I.keys[i];
        if ((k & hmask) == prefix) atomicAdd(&s_hist[(k >> shift) & 255u], 1u);
      }
      __syncthreads();
      if (tid < 32) {                            // warp 0: lane l owns bins 8l .. 8l+7
        unsigned int c[8], sum = 0u;
#pragma unroll
        for (int j = 0; j < 8; j++) { c[j] = s_hist[8 * tid + j]; sum += c[j]; }
        unsigned int incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned int v = __shfl_up_sync(0xffffffffu, incl, o);
          if (tid >= o) incl += v;
        }
        const unsigned int excl = incl - sum;
        if (excl < need && need <= incl) {       // exactly one lane holds the digit
          unsigned int acc = excl;
          int d = 8 * tid + 7;
#pragma unroll
          for (int j = 0; j < 8; j++) {
            if (acc + c[j] >= need) { d = 8 * tid + j; break; }
            acc += c[j];
          }
          s_prefix = prefix | ((unsigned)d << shift);
          s_need = need - acc;
        }
      }
      __syncthreads();
      prefix = s_prefix;
      need = s_need;
    }
    thr = prefix;
  }

  if (tid == 0) s_count = 0u;
  __syncthreads();
  for (int i = tid; i < n; i += RK_SELECT_THREADS) {
    const unsigned int k = I.keys[i];
    if (k <= thr) {
      const unsigned int pos = atomicAdd(&s_count, 1u);
      const SiftPoint *q = I.in + i;
      unsigned int *d = I.sk + pos;
      d[0] = k;
      d[(size_t)1 * P.maxIn] = ord_key(q->subsampling);
      d[(size_t)2 * P.maxIn] = ord_key(q->ypos);
      d[(size_t)3 * P.maxIn] = ord_key(q->xpos);
      d[(size_t)4 * P.maxIn] = ord_key(q->scale);
      d[(size_t)5 * P.maxIn] = ord_key(q->orientation);
      d[(size_t)6 * P.maxIn] = (unsigned)i;
      I.rank[pos] = 0u;
    }
  }
  __syncthreads();
  if (tid == 0) {
    I.nsurv[0] = s_count;
    I.cnt[2] = (unsigned)keep;                   // the output count, brought back with the counters
  }
}

// a < b on (k1 .. k5, candidate index) for keys equal on k0; the index only separates records equal on all six
// fields, which the extractor never produces
__device__ __forceinline__ bool rank_tail_less(const unsigned int (&a)[RK_KEY_WORDS + 1], const unsigned int (&b)[RK_KEY_WORDS + 1])
{
#pragma unroll
  for (int w = 1; w <= RK_KEY_WORDS; w++)
    if (a[w] != b[w]) return a[w] < b[w];
  return false;
}

__global__ void __launch_bounds__(RK_ORDER_THREADS) rank_order_kernel(const __grid_constant__ RankParams P)
{
  __shared__ unsigned int s_k[RK_KEY_WORDS + 1][RK_ORDER_THREADS];
  const int tid = threadIdx.x;
  const RankImage I = rank_image(P, blockIdx.z);
  const int S = (int)I.nsurv[0];
  for (int base = blockIdx.x * RK_ORDER_THREADS; base < S; base += gridDim.x * RK_ORDER_THREADS) {
    const int i = base + tid;
    const bool valid = i < S;
    unsigned int mine[RK_KEY_WORDS + 1];
#pragma unroll
    for (int w = 0; w <= RK_KEY_WORDS; w++) mine[w] = valid ? I.sk[(size_t)w * P.maxIn + i] : 0xffffffffu;
    int rank = 0;
    for (int t0 = blockIdx.y * RK_ORDER_THREADS; t0 < S; t0 += gridDim.y * RK_ORDER_THREADS) {
      __syncthreads();
      if (t0 + tid < S)
#pragma unroll
        for (int w = 0; w <= RK_KEY_WORDS; w++) s_k[w][tid] = I.sk[(size_t)w * P.maxIn + t0 + tid];
      __syncthreads();
      const int m = min(RK_ORDER_THREADS, S - t0);
      if (valid) {
#pragma unroll 4
        for (int j = 0; j < m; j++) {
          const unsigned int a = s_k[0][j];
          if (a < mine[0]) rank++;
          else if (a == mine[0]) {               // equal |sharpness|: primary/secondary pairs and repeated values
            unsigned int other[RK_KEY_WORDS + 1];
#pragma unroll
            for (int w = 0; w <= RK_KEY_WORDS; w++) other[w] = s_k[w][j];
            if (rank_tail_less(other, mine)) rank++;
          }
        }
      }
    }
    if (valid && rank > 0) atomicAdd(&I.rank[i], (unsigned)rank);
  }
}

__global__ void __launch_bounds__(RK_GATHER_THREADS) rank_gather_kernel(const __grid_constant__ RankParams P)
{
  constexpr int V = (int)(sizeof(SiftPoint) / sizeof(uint4));   // 36
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = RK_GATHER_THREADS / 32;
  const RankImage I = rank_image(P, blockIdx.y);
  const int S = (int)I.nsurv[0];
  const unsigned int keep = I.cnt[2];
  // describe places secondary orientations after the primaries and leaves their empty[0] (the detector's cap
  // bookkeeping tag, bytes 52..55) unwritten: it is cleared so that the output depends on the keypoints alone
  const unsigned int numPrim = min(I.cnt[0], (unsigned)P.maxIn);
  for (int i = blockIdx.x * warps + warp; i < S; i += gridDim.x * warps) {
    const unsigned int r = I.rank[i];
    if (r >= keep) continue;
    const unsigned int idx = I.sk[(size_t)RK_KEY_WORDS * P.maxIn + i];
    const uint4 *__restrict__ src = reinterpret_cast<const uint4 *>(I.in + idx);
    uint4 *__restrict__ dst = reinterpret_cast<uint4 *>(I.out + r);
    uint4 a = src[lane];
    uint4 b;
    if (lane < V - 32) b = src[32 + lane];
    if (lane == 3 && idx >= numPrim) a.y = 0u;
    dst[lane] = a;
    if (lane < V - 32) dst[32 + lane] = b;
  }
}

int launch_rank(const RankParams &p, int batch, int sms, cudaStream_t st)
{
  if (batch < 1 || p.maxIn < 1 || p.maxOut < 1 || p.maxIn > CS_RANK_MAX_IN) {
    set_error("rank: bad batch %d or capacities %d / %d", batch, p.maxIn, p.maxOut);
    return CS_E_ARG;
  }
  rank_select_kernel<<<batch, RK_SELECT_THREADS, 0, st>>>(p);
  count_launch();
  CS_CUDA(cudaGetLastError());
  // survivors number at most maxIn: oc x oc CTAs per image (tiles of ranked x tiles compared, grid-stride beyond),
  // about 8 CTAs per SM over the batch
  int ox = idivup(p.maxIn, RK_ORDER_THREADS), oc = (int)sqrtf((float)(8 * sms / batch));
  if (oc < 4) oc = 4;
  if (ox > oc) ox = oc;
  rank_order_kernel<<<dim3(ox, ox, batch), RK_ORDER_THREADS, 0, st>>>(p);
  count_launch();
  CS_CUDA(cudaGetLastError());
  int gx = idivup(p.maxIn, RK_GATHER_THREADS / 32), gc = 4 * sms / batch;
  if (gc < 4) gc = 4;
  if (gx > gc) gx = gc;
  rank_gather_kernel<<<dim3(gx, batch), RK_GATHER_THREADS, 0, st>>>(p);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace cs
