// detect2.cu -- marching detector: 8-scale blur + DoG + 3x3x3 extrema + sub-pixel refinement, all octaves of
// a whole BATCH of images in one launch (detect3_kernel).
//
// Behavioural spec: reference LaplaceMultiMem (cudaSiftD.cu:1753-1793, host :460-487) and
// FindPointsMultiNew (cudaSiftD.cu:1292-1431, host :489-514).  Per-pixel arithmetic and refinement from
// sift_arith.cuh (pinned to the reference's SASS: which products are fused, the order of the sums), new dataflow:
//
//  * A work item is a column strip (256 staged columns -> 248 DoG columns -> 244 tested columns) times a
//    range of rows of one octave of one image.  The CTA marches down the rows; nothing is recomputed
//    vertically: the 9-row window of every column lives in REGISTERS and slides by one row per step.
//  * FP32 pairs (tma.cuh): the two halves of every register pair are two ROW STREAMS of the same item
//    (row y and row y + hs), so all horizontal neighbours are whole aligned pairs.
//  * Input rows arrive by TMA (cp.async.bulk.tensor.2d, one 256x1 box per row and stream, row index clamped
//    by the issuing thread, columns clamped by the reading thread) into an 8-deep ring -> no address
//    arithmetic and no global loads in the loop.
//  * Warp-specialised, one CTA of 20 warps per SM (five warpgroups):
//      warps 12-19 (producers, two warpgroups): vertical pass of all 8 scales (thread = one staged column: warps 12-15
//                              take columns 0-127, warps 16-19 columns 128-255; 9-row register window, 40 taps in
//                              registers) and the TMA row ring (one lane issues it) -- a serial path, kept short so
//                              that the consumer groups, not the producers, set the pace; results go to shared memory
//                              once (STS.64)
//      warps 0-3 / 4-7 / 8-11 (consumer groups 0 / 1 / 2): horizontal pass + DoG + candidate flags of the steps
//                              k = g mod 3 (2 x 16 column groups), then the extrema tests of row k-4; each group has
//                              three steps of time for one step of work.  Lane = (scale, 8 columns): 8 conflict-free
//                              LDS.128 fetch the 16 pairs, the DoG difference takes the neighbouring scale from the
//                              neighbouring lane (shuffle), the DoG row goes to an 8-deep ring in shared memory.
//  * |DoG| > thresh is decided on the register copies; flagged (pixel, plane) candidates are listed and tested
//    four steps later, when the rows above and below exist.
//
// The producers run ahead of the consumers through three vertical-result buffers (buffer = group); hand-over is by
// named barriers (bar.arrive / bar.sync) instead of CTA-wide barriers.  Each of them counts the 256 producer threads
// and the 128 threads of one group, so it completes only when every thread of both producer warpgroups has arrived:
// the producers pass them together, and every statement below about "the producers" holds for all 256.
//   FULL[g]  producers -> group g: v[g] written        EMPTY[g] group g -> producers: v[g] is in registers
//   DONE[g]  group g -> producers: the DoG row and the candidate list of its step are written (the extrema tests of
//            an older row follow, off the producers' critical path)
//   LATE[g]  group g -> producers: its previous step is complete, tests included (signalled at the start of the next step)
//            The producers check DONE of step m-3 and LATE of step m-4 just before they signal FULL of step m.  Hence,
//            when a group passes FULL of step k, every DoG row <= k-3 is written and every step <= k-4 of every group
//            is complete: it may test the extrema of row k-4 (rows k-5..k-3) and overwrite ring slot k mod 8 (last
//            read for rows k-9..k-7 in steps k-5, k-4 and -- by this same group -- k-3).
//
// Shared memory per row pair and step: 128 (vertical STS) + 256 (horizontal LDS) + 128 (shuffles) + 112 (DoG
// STS) wavefronts for 2 x 244 pixels x 8 scales = 1.3 wavefronts per pixel (detect.cu: 2.7).
#include "common.cuh"
#include "sift_arith.cuh"

namespace cs {

#define D2_IW 256            // staged input columns per strip (one TMA box row)
#define D2_TESTED CS_D2_STRIP // tested DoG columns per strip: 1..244 (DoG column d <-> input column d + 4); a multiple of 4,
                             // because TMA wants the first column of a box (x0 - 4) on a 16-byte boundary
#define D2_NS 8              // input ring depth (row pairs)
#define D2_VROW2 258         // float2 per (scale) row of vertical results: 256 + one 16-byte pad
#define D2_VBUF2 (8 * D2_VROW2)
#define D2_RROWF 500         // floats per DoG plane row in the ring: 248 pairs + one 16-byte pad
#define D2_RSLOTF (7 * D2_RROWF)
#define D2_LCAP 510          // candidate list capacity per step (more: the step is scanned exhaustively)
#define D2_KQ 32             // keypoints parked per item before the slots are allocated
#define D2_SMEM_IN (D2_NS * 2 * D2_IW * 4)            // 16384

struct D2Keypoint { float x, y, scale, sharpness, edgeness, subsampling; unsigned int tag; };

// powf(2.0f, scale / 5) of cudaSiftD.cu:1417 for the five scales an extremum can have.  The table is filled on the
// device by the same powf (d2_fill_pow_table, first launch per device), so the values are the ones the reference's
// expression yields; it takes ~100 instructions out of the refinement of every extremum.
__device__ float d2_pow_table[CS_NUM_SCALES];
__global__ void d2_fill_pow_table()
{
  if (threadIdx.x < CS_NUM_SCALES) d2_pow_table[threadIdx.x] = powf(2.0f, __fdiv_rn((float)threadIdx.x, (float)CS_NUM_SCALES));
}

__device__ __forceinline__ void d2_store_keypoint(SiftPoint *pts, int maxPts, unsigned int idx, const D2Keypoint &kp)
{
  if (idx >= (unsigned)maxPts) idx = maxPts - 1;    // cudaSiftD.cu:1421
  SiftPoint *q = pts + idx;
  q->xpos = kp.x;
  q->ypos = kp.y;
  q->scale = kp.scale;
  q->sharpness = kp.sharpness;
  q->edgeness = kp.edgeness;
  q->subsampling = kp.subsampling;
  q->empty[0] = __uint_as_float(kp.tag);            // integer position of the extremum (cap32 bookkeeping)
}

// cudaSiftD.cu:1383-1429 (sift_arith.cuh).  v[p][dy][dx]: the 3x3x3 DoG neighbourhood, candidate at [1][1][1].
__device__ __forceinline__ void d2_refine(const float (&v)[3][3][3], int gx, int gy, int scale, float subsampling,
                                       float lowestScale, float edgeLimit, float factor, unsigned int tag,
                                       D2Keypoint *s_kq, int *s_kn, SiftPoint *pts, unsigned int *counter, int maxPts)
{
  D2Keypoint kp;
  if (!refine_extremum(v, gx, gy, edgeLimit, factor, lowestScale, [&] { return d2_pow_table[scale]; }, kp)) return;
  kp.subsampling = subsampling;
  kp.tag = tag;
  const int q = atomicAdd(s_kn, 1);
  if (q < D2_KQ) s_kq[q] = kp;
  else d2_store_keypoint(pts, maxPts, atomicAdd(counter, 1u), kp);
}

#define D3_GT 128                                        // threads per consumer group (one warpgroup)
#define D3_PT 256                                        // producer threads (two warpgroups), one staged column each
// 640 threads leave 96 registers per thread.  Both roles fit without a setmaxnreg rebalance: in the sm_90a SASS the
// consumer code peaks at 94 registers and the one-column producer code at 60, with no spills.
#define D3_THREADS (3 * D3_GT + D3_PT)
#define D3_HAND (D3_GT + D3_PT)                          // threads on a FULL / EMPTY / DONE / LATE barrier
#define D3_RS 8
#define D3_SMEM_RING (D3_RS * D2_RSLOTF * 4)            // 112000
#define D3_SMEM_LIST (D3_RS * 512 * 2)                  // 8192
#define D3_NB 3                                          // vertical-result buffers
#define D3_SMEM_V (D3_NB * D2_VBUF2 * 8)                // 49536
#define D3_SMEM_BYTES (D2_SMEM_IN + D3_SMEM_V + D3_SMEM_RING + D3_SMEM_LIST)   // 186112

__device__ __forceinline__ void nb_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void nb_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
#define NB_FULL 1      // + group (3)
#define NB_EMPTY 4     // + group (3)
#define NB_DONE 7      // + group (3)
#define NB_PINT 10
#define NB_LATE 11     // + group (3)

struct D3Item {
  int level, img, x0, ry0, hs, w, h;
  float thresh, subsampling, lowestScale, edgeLimit, factor;
  SiftPoint *pts;
  unsigned int *counters;
  int maxPts;
  unsigned int *cells;
  int cellBase, cellsX, capLimit;
};

// Extrema of step j (DoG rows ry0-1+j / ry0+hs-1+j) by the 128 threads of a consumer group; rows j-1, j, j+1 are
// complete.
__device__ __forceinline__ void d3_extrema(const D3Item &I, int j, int pt, const float *s_ring,
                                           const unsigned short *s_list, const int *s_cnt, D2Keypoint *s_kq, int *s_kn)
{
  const int qj = j & (D3_RS - 1);
  int n = s_cnt[qj];
  if (n == 0) return;
  const bool scan = n > D2_LCAP;                    // list overflow: test every pixel of the row pair
  if (scan) n = 2 * CS_NUM_SCALES * D2_TESTED;
  const float *rm = s_ring + ((j + D3_RS - 1) & (D3_RS - 1)) * D2_RSLOTF, *r0 = s_ring + qj * D2_RSLOTF,
              *rp = s_ring + ((j + 1) & (D3_RS - 1)) * D2_RSLOTF;
  for (int i = pt; i < n; i += D3_GT) {
    int dc, p, hf;
    if (!scan) {
      const int e = s_list[qj * 512 + i];
      dc = e & 255; p = (e >> 8) & 7; hf = e >> 11;
    } else {
      hf = i / (CS_NUM_SCALES * D2_TESTED);
      const int r = i - hf * (CS_NUM_SCALES * D2_TESTED);
      p = r / D2_TESTED;
      dc = 1 + r - p * D2_TESTED;
      p += 1;
      const int gy_ = (hf ? I.ry0 + I.hs - 1 : I.ry0 - 1) + j;
      if (gy_ > I.h - 2 || I.x0 + dc > I.w - 2) continue;
    }
    const int o = p * D2_RROWF + 2 * dc + hf;
    const float c = r0[o];
    if (!(fabsf(c) > I.thresh)) continue;
    // the strict 26-neighbour test of cudaSiftD.cu:1340-1358 in two stages (the outcome is the same): the 8 neighbours
    // in the candidate's own plane first -- most candidates fail there, and the other 18 values are never loaded
    float v[3][3][3];
    bool mx = true, mn = true;
#pragma unroll
    for (int dx = 0; dx < 3; dx++) {
      const int oo = o + 2 * (dx - 1);
      v[1][0][dx] = rm[oo];
      v[1][1][dx] = r0[oo];
      v[1][2][dx] = rp[oo];
    }
#pragma unroll
    for (int dy = 0; dy < 3; dy++)
#pragma unroll
      for (int dx = 0; dx < 3; dx++)
        if (dy != 1 || dx != 1) { mx = mx && (c > v[1][dy][dx]); mn = mn && (c < v[1][dy][dx]); }
    if (!(c > 0.0f ? mx : mn)) continue;
#pragma unroll
    for (int pp = 0; pp < 3; pp += 2)
#pragma unroll
      for (int dx = 0; dx < 3; dx++) {
        const int oo = o + (pp - 1) * D2_RROWF + 2 * (dx - 1);
        v[pp][0][dx] = rm[oo];
        v[pp][1][dx] = r0[oo];
        v[pp][2][dx] = rp[oo];
      }
#pragma unroll
    for (int pp = 0; pp < 3; pp += 2)
#pragma unroll
      for (int dy = 0; dy < 3; dy++)
#pragma unroll
        for (int dx = 0; dx < 3; dx++) { mx = mx && (c > v[pp][dy][dx]); mn = mn && (c < v[pp][dy][dx]); }
    if (c > 0.0f ? mx : mn) {
      const int gx = I.x0 + dc, gy = (hf ? I.ry0 + I.hs - 1 : I.ry0 - 1) + j;
      const unsigned int tag = (unsigned)gx | ((unsigned)gy << 13) | ((unsigned)(p - 1) << 26) | ((unsigned)I.level << 29);
      if (I.cells) {                                // extrema per 30x8 block and scale (reference cap, cudaSiftD.cu:1371)
        const int cell = I.cellBase + ((gy >> 3) * I.cellsX + gx / 30) * CS_NUM_SCALES + (p - 1);
        // no return value -> RED: the count is not on this thread's critical path; the fix-up kernel finds the
        // cells that went past the limit by scanning the counters
        atomicAdd(I.cells + (cell >> 2), 1u << (8 * (cell & 3)));
      }
      d2_refine(v, gx, gy, p - 1, I.subsampling, I.lowestScale, I.edgeLimit, I.factor, tag, s_kq, s_kn, I.pts,
                &I.counters[0], I.maxPts);
    }
  }
}

// vertical pass of one step, all 8 scales of the thread's column
template <int PH>
__device__ __forceinline__ void d3_vertical(f32x2 (&W)[9], f32x2 n, const float (&kv)[CS_LAPLACE_S][5], float2 *vdst)
{
#define D3_WI(i) ((PH + 1 + (i)) % 9)
  W[PH] = n;
  const f32x2 c = W[D3_WI(4)];
  const f32x2 p1 = add2(W[D3_WI(3)], W[D3_WI(5)]), p2 = add2(W[D3_WI(2)], W[D3_WI(6)]);
  const f32x2 p3 = add2(W[D3_WI(1)], W[D3_WI(7)]), p4 = add2(W[D3_WI(0)], W[D3_WI(8)]);
#pragma unroll
  for (int s = 0; s < CS_LAPLACE_S; s++) vdst[s * D2_VROW2] = upk(laplace9(kv[s], c, p1, p2, p3, p4));
#undef D3_WI
}

__global__ void __launch_bounds__(D3_THREADS, 1)
detect3_kernel(const __grid_constant__ Detect2Params P)
{
  extern __shared__ __align__(128) unsigned char d2_smem[];
  float *s_in = reinterpret_cast<float *>(d2_smem);                                         // [slot][stream][256]
  float2 *s_v = reinterpret_cast<float2 *>(d2_smem + D2_SMEM_IN);                           // [buf][scale][258]
  float *s_ring = reinterpret_cast<float *>(d2_smem + D2_SMEM_IN + D3_SMEM_V);              // [slot][plane][500]
  unsigned short *s_list = reinterpret_cast<unsigned short *>(d2_smem + D2_SMEM_IN + D3_SMEM_V + D3_SMEM_RING);
  __shared__ __align__(8) uint64_t s_full[D2_NS];
  __shared__ int s_cnt[D3_RS];
  __shared__ int s_kn, s_next;
  __shared__ D2Keypoint s_kq[D2_KQ];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool producer = warp >= 12;       // the highest warp ids: the issue arbiter favours them
  const int pt = tid - 3 * D3_GT;         // producer thread index (0..255) = staged column

  int item = blockIdx.x;
  unsigned int req = 0;
  if (tid == 0) req = gridDim.x + atomicAdd(P.sched, 1u);

  while (item < P.numItems) {
    const uint4 it = __ldg(P.items + item);
    const int level = it.x & 0xff, img = it.x >> 8;
    const int x0 = (int)it.y, ry0 = (int)it.z, hs = (int)it.w;
    const D2Level &L = P.lev[level];
    const int w = L.w, h = L.h;
    const int nsteps = hs + 2;                            // DoG rows ry0-1+k (stream A), ry0+hs-1+k (stream B), k < nsteps
    const int nrows = 8 + nsteps;                         // input rows per stream: ry0-5+i (A), i < nrows

    __syncthreads();     // previous item complete (extrema, keypoint flush)
    if (tid == 0) {
      for (int i = 0; i < D2_NS; i++) mbarrier_init(&s_full[i], 1);
      mbarrier_init_fence();
      for (int i = 0; i < D3_RS; i++) s_cnt[i] = 0;
      s_kn = 0;
      s_next = (int)req;                                  // requested during the previous item
      req = gridDim.x + atomicAdd(P.sched, 1u);
    }
    __syncthreads();

    if (producer) {
      // ================================================================== producers
      const CUtensorMap *map = P.maps + (size_t)img * CS_MAX_LEVELS + level;
      if (pt == 0) {
        tensormap_acquire(map);
        for (int i = 0; i < D2_NS; i++) {                 // prologue rows: all in flight at once
          mbarrier_expect_tx(&s_full[i], 2 * D2_IW * 4);
          tma_load_2d(s_in + (2 * i) * D2_IW, map, x0 - 4, min(max(ry0 - 5 + i, 0), h - 1), &s_full[i]);
          tma_load_2d(s_in + (2 * i + 1) * D2_IW, map, x0 - 4, min(max(ry0 + hs - 5 + i, 0), h - 1), &s_full[i]);
        }
      }
      // the column this thread reads from a staged row (clamped to the image: cudaSiftD.cu:1764-1767)
      const int ci = min(max(x0 - 4 + pt, 0), w - 1) - (x0 - 4);
      float kv[CS_LAPLACE_S][5];
#pragma unroll
      for (int s = 0; s < CS_LAPLACE_S; s++)
#pragma unroll
        for (int j = 0; j < 5; j++) kv[s][j] = L.taps.k[s][j];
      f32x2 W[9];
#pragma unroll
      for (int i = 0; i < 8; i++) {
        mbarrier_wait(&s_full[i], 0);
        const float *ra = s_in + (2 * i) * D2_IW, *rb = ra + D2_IW;
        W[i] = pk2(ra[ci], rb[ci]);
      }
      W[8] = 0ull;
      nb_sync(NB_PINT, D3_PT);                            // every producer has read the prologue rows
      if (pt == 0) {
        for (int i = 0; i < D2_NS; i++)
          if (8 + i < nrows) {
            mbarrier_expect_tx(&s_full[i], 2 * D2_IW * 4);
            tma_load_2d(s_in + (2 * i) * D2_IW, map, x0 - 4, min(max(ry0 + 3 + i, 0), h - 1), &s_full[i]);
            tma_load_2d(s_in + (2 * i + 1) * D2_IW, map, x0 - 4, min(max(ry0 + hs + 3 + i, 0), h - 1), &s_full[i]);
          }
      }
      // rows of step 0 (software pipelining: the rows of step m+1 are fetched at the end of step m)
      f32x2 n;
      {
        mbarrier_wait(&s_full[0], 1);
        n = pk2(s_in[ci], s_in[D2_IW + ci]);
      }
      // step m: window slot of the newest row = (8 + m) % 9 -> unrolled by 9 so that the slots are compile-time.
      // The EMPTY hand-over doubles as the producers' own barrier: it completes only when all 256 producer threads
      // (both warpgroups) have arrived, so past it every producer has finished step m-1, and the input slots read up to
      // then may be refilled.
#define D3_PSTEP(p)                                                                                           \
  {                                                                                                           \
    const int m = m0 + (p);                                                                                   \
    if (m >= nsteps + 3) break;                                                                               \
    f32x2 xn = 0ull;                                                                                          \
    if (m < nsteps) {                                                                                         \
      if (m >= D3_NB) nb_sync(NB_EMPTY + (p) % D3_NB, D3_HAND);                                               \
      if (m + 1 < nsteps) {                  /* rows of step m+1: their latency hides behind this step's math */ \
        const int slot = (m + 1) & (D2_NS - 1);                                                               \
        mbarrier_wait(&s_full[slot], ((9 + m) >> 3) & 1);                                                     \
        const float *ra = s_in + (2 * slot) * D2_IW, *rb = ra + D2_IW;                                        \
        xn = pk2(ra[ci], rb[ci]);                                                                             \
      }                                                                                                       \
      d3_vertical<(8 + (p)) % 9>(W, n, kv, s_v + ((p) % D3_NB) * D2_VBUF2 + pt);                              \
      n = xn;                                                                                                 \
    }                                                                                                         \
    /* DONE: the group's previous step (m-3) has written its DoG row and candidate list.  LATE: step m-4 (another */ \
    /* group) is complete including its extrema tests (rows m-9..m-7, list of row m-8) */                     \
    if (m >= D3_NB) nb_sync(NB_DONE + (p) % D3_NB, D3_HAND);                                                  \
    if (m >= D3_NB + 1) nb_sync(NB_LATE + ((p) + 2) % D3_NB, D3_HAND);                                        \
    if (pt == 0 && m >= 8) s_cnt[m & (D3_RS - 1)] = 0;           /* list of row m-8: used again by step m */    \
    nb_arrive(NB_FULL + (p) % D3_NB, D3_HAND);                 /* in the drain steps: only releases the tests */ \
    if (pt == 0 && m >= D3_NB && m < nsteps) {                                                                \
      /* past EMPTY of this step every producer has finished step m-1: refill the slots read up to then */     \
      for (int r = (m == D3_NB ? 0 : m - 1); r < m; r++)                                                      \
        if (16 + r < nrows) {                                                                                 \
          const int rs = r & (D2_NS - 1);                                                                     \
          mbarrier_expect_tx(&s_full[rs], 2 * D2_IW * 4);                                                     \
          tma_load_2d(s_in + (2 * rs) * D2_IW, map, x0 - 4, min(max(ry0 + 11 + r, 0), h - 1), &s_full[rs]);     \
          tma_load_2d(s_in + (2 * rs + 1) * D2_IW, map, x0 - 4, min(max(ry0 + hs + 11 + r, 0), h - 1), &s_full[rs]); \
        }                                                                                                     \
    }                                                                                                         \
  }
      for (int m0 = 0;; m0 += 9) {
        D3_PSTEP(0) D3_PSTEP(1) D3_PSTEP(2) D3_PSTEP(3) D3_PSTEP(4) D3_PSTEP(5) D3_PSTEP(6) D3_PSTEP(7) D3_PSTEP(8)
      }
#undef D3_PSTEP
    } else {
      // ================================================================== consumers
      // No divergence in here: lanes whose 8 columns lie outside the strip or the image compute on whatever the
      // buffer holds (in-bounds garbage) and only their stores and candidate flags are masked, so the shuffles
      // run with the full mask and every shared address is (per-thread constant) + (per-step constant).
      const int g = warp >> 2, wg = warp & 3;                   // group g: steps k = g mod 3, buffer g
      const int hs_ = lane & 7, cgl = lane >> 3;                // scale, column group within the warp
      const float thresh = P.thresh;
      float kh[5];
#pragma unroll
      for (int j = 0; j < 5; j++) kh[j] = L.taps.k[hs_][j];
      const float4 *vsrc0 = reinterpret_cast<const float4 *>(s_v + g * D2_VBUF2 + hs_ * D2_VROW2 + 8 * (4 * wg + cgl));
      float *rdst0 = s_ring + max(hs_ - 1, 0) * D2_RROWF + 16 * (4 * wg + cgl);
      D3Item I;
      I.level = level; I.img = img; I.x0 = x0; I.ry0 = ry0; I.hs = hs; I.w = w; I.h = h;
      I.thresh = P.thresh; I.subsampling = L.subsampling; I.lowestScale = L.lowestScale;
      I.edgeLimit = P.edgeLimit; I.factor = P.factor;
      I.pts = P.pts + (size_t)img * P.ptsStride;
      I.counters = P.counters + (size_t)img * CS_CNT_STRIDE;
      I.maxPts = P.maxPts;
      I.cells = P.cells ? P.cells + (size_t)img * P.cellWords : nullptr;
      I.cellBase = P.cellBase[level]; I.cellsX = P.cellsX[level]; I.capLimit = P.capLimit;
      const bool testable = hs_ >= 2 && hs_ <= 6;               // DoG planes 1..5
      const int tig = tid & 127;                                // thread index within the group
      // columns of the lane's 8 that are tested (bits d and 8 + d for the two streams), per pass: fixed for the item
      unsigned colok[2];
#pragma unroll
      for (int pass = 0; pass < 2; pass++) {
        colok[pass] = 0;
#pragma unroll
        for (int d = 0; d < 8; d++) {
          const int dc = 8 * (16 * pass + 4 * wg + cgl) + d;
          if (dc >= 1 && dc <= D2_TESTED && x0 + dc <= w - 2) colok[pass] |= 0x101u << d;
        }
      }
      for (int k = g; k < nsteps + 3; k += D3_NB) {
        const int q = k & (D3_RS - 1);
        // LATE: this group's previous step (k-3) is complete, extrema tests included.  It is signalled here, after the
        // group has passed FULL of step k, and not at the end of step k-3: the producers consume it at their step k+1,
        // which is before they can signal FULL of step k+3, so two arrivals never pile up on the barrier.
        const bool late = k >= D3_NB && k - D3_NB <= nsteps - 2;
        if (k >= nsteps) {                                      // drain: only the extrema of the last rows
          nb_sync(NB_FULL + g, D3_HAND);
          if (late) nb_arrive(NB_LATE + g, D3_HAND);
          if (k - 4 <= hs && s_cnt[(k - 4) & (D3_RS - 1)] != 0) d3_extrema(I, k - 4, tig, s_ring, s_list, s_cnt, s_kq, &s_kn);
          continue;
        }
        const bool rowsTested = testable && k >= 1 && k <= hs;
        const unsigned rowok = (ry0 - 1 + k <= h - 2 ? 0xffu : 0u) | (ry0 + hs - 1 + k <= h - 2 ? 0xff00u : 0u);
        nb_sync(NB_FULL + g, D3_HAND);
        if (late) nb_arrive(NB_LATE + g, D3_HAND);
#pragma unroll
        for (int pass = 0; pass < 2; pass++) {
          const int cg = 16 * pass + 4 * wg + cgl;
          const bool act = cg < 31 && x0 + 8 * cg <= w - 1;      // this lane's 8 DoG columns start inside the image
          const float4 *src = vsrc0 + 64 * pass;                 // 16 column groups further = 128 pairs
          f32x2 V[16];
#pragma unroll
          for (int j = 0; j < 8; j++) {
            const float4 t4 = src[j];
            V[2 * j] = pk2(t4.x, t4.y);
            V[2 * j + 1] = pk2(t4.z, t4.w);
          }
          if (pass == 1 && k + D3_NB < nsteps) nb_arrive(NB_EMPTY + g, D3_HAND);   // v[g] is in registers
          f32x2 dg[8];
#pragma unroll
          for (int d = 0; d < 8; d++) {
            const f32x2 o = laplace9(kh, V[d + 4], add2(V[d + 3], V[d + 5]), add2(V[d + 2], V[d + 6]),
                                     add2(V[d + 1], V[d + 7]), add2(V[d], V[d + 8]));
            const float2 of = upk(o);
            const float plo = __shfl_up_sync(0xffffffffu, of.x, 1), phi = __shfl_up_sync(0xffffffffu, of.y, 1);
            dg[d] = sub2(o, pk2(plo, phi));                 // blur[s] - blur[s-1]: DoG plane s-1 (cudaSiftD.cu:1790)
          }
          if (act && hs_ >= 1) {
            float4 *dst = reinterpret_cast<float4 *>(rdst0 + q * D2_RSLOTF + 256 * pass);
#pragma unroll
            for (int j = 0; j < 4; j++) {
              const float2 a = upk(dg[2 * j]), b = upk(dg[2 * j + 1]);
              dst[j] = make_float4(a.x, a.y, b.x, b.y);
            }
          }
          float m = 0.0f;
#pragma unroll
          for (int d = 0; d < 8; d++) {
            const float2 a = upk(dg[d]);
            m = fmaxf(m, fmaxf(fabsf(a.x), fabsf(a.y)));
          }
          if (m > thresh && rowsTested && act) {
            unsigned bits = 0;
#pragma unroll
            for (int d = 0; d < 8; d++) {
              const float2 a = upk(dg[d]);
              // a necessary condition that is already in registers: an extremum beats its left and right neighbours
              // (columns 1..6 of the lane's 8; the two outer columns are decided by the full test)
              bool ex = true, ey = true;
              if (d >= 1 && d <= 6) {
                const float2 l = upk(dg[d - 1]), r = upk(dg[d + 1]);
                ex = a.x > 0.0f ? (a.x > l.x && a.x > r.x) : (a.x < l.x && a.x < r.x);
                ey = a.y > 0.0f ? (a.y > l.y && a.y > r.y) : (a.y < l.y && a.y < r.y);
              }
              if (ex && fabsf(a.x) > thresh) bits |= 1u << d;
              if (ey && fabsf(a.y) > thresh) bits |= 0x100u << d;
            }
            bits &= colok[pass] & rowok;
            if (bits) {
              int at = atomicAdd(&s_cnt[q], __popc(bits));
              while (bits) {
                const int b = __ffs(bits) - 1;
                bits &= bits - 1;
                if (at < D2_LCAP) s_list[q * 512 + at] = (unsigned short)((8 * cg + (b & 7)) | ((hs_ - 1) << 8) | ((b >> 3) << 11));
                at++;
              }
            }
          }
        }
        nb_arrive(NB_DONE + g, D3_HAND);                       // row k and its candidate list are written
        // rows k-5..k-3 are complete; the tests run only when the row has candidates at all
        if (k >= 5 && s_cnt[(k - 4) & (D3_RS - 1)] != 0) d3_extrema(I, k - 4, tig, s_ring, s_list, s_cnt, s_kq, &s_kn);
      }
    }
    __syncthreads();
    {
      const int nkq = min(s_kn, D2_KQ);
      if (tid < nkq)
        d2_store_keypoint(P.pts + (size_t)img * P.ptsStride, P.maxPts,
                          atomicAdd(&P.counters[(size_t)img * CS_CNT_STRIDE], 1u), s_kq[tid]);
    }
    item = s_next;
  }
}


// once per device, outside any stream capture (Pipeline::init)
static int g_d2_table[64];
int detect2_init_device()
{
  int dev = 0;
  CS_CUDA(cudaGetDevice(&dev));
  if (dev < 64 && g_d2_table[dev]) return 0;
  d2_fill_pow_table<<<1, 32>>>();
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaDeviceSynchronize());
  if (dev < 64) g_d2_table[dev] = 1;
  return 0;
}

static int g_d2_configured[64];

int launch_detect2(const Detect2Params &p, int sms, cudaStream_t st)
{
  if (p.numItems <= 0) return 0;
  int dev = 0;
  CS_CUDA(cudaGetDevice(&dev));
  if (dev < 64 && !g_d2_configured[dev]) {      // per device: cudaFuncSetAttribute applies to the current device only
    CS_CUDA(cudaFuncSetAttribute(detect3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, D3_SMEM_BYTES));
    g_d2_configured[dev] = 1;
  }
  const int grid = p.numItems < sms ? p.numItems : sms;
  detect3_kernel<<<grid, D3_THREADS, D3_SMEM_BYTES, st>>>(p);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace cs
