// cap32.cu -- the reference's cap of 32 extrema per (30x8 block, scale) (quirk of FindPointsMultiNew,
// cudaSiftD.cu:1361-1380: `pos<MEMWID` keeps the first 32 in (column, row) order, `tx<totbits` refines them).
//
// The detector (detect2.cu) counts the extrema of every such cell in packed 8-bit counters (reductions without a
// return value); this kernel scans the counters for cells past the limit.  That almost never happens (it needs > 13 %
// of a block's pixels to be 26-neighbour extrema above the threshold), so the repair is a separate, tiny, usually empty
// kernel: per listed cell it recomputes the cell's DoG planes from the octave base image with the detector's arithmetic
// (sift_arith.cuh), ranks the extrema in the reference's order and deletes the keypoints of rank >= 32 from the image's
// list (those that survived refinement; the list is unordered anyway, so a hole is filled with the last record).
#include "common.cuh"
#include "sift_arith.cuh"

namespace cs {

#define C32_THREADS 256
#define C32_W 32              // DoG columns: cell column -1 .. +30
#define C32_H 10              // DoG rows: cell row -1 .. +8
#define C32_VW (C32_W + 8)    // columns of vertical results

__global__ void __launch_bounds__(C32_THREADS)
cap32_fixup_kernel(const __grid_constant__ Detect2Params P)
{
  const int img = blockIdx.x, tid = threadIdx.x;
  unsigned int *counters = P.counters + (size_t)img * CS_CNT_STRIDE;
  // the cells that received more than capLimit extrema: scan the image's packed 8-bit counters (the detector only
  // counts, with fire-and-forget reductions)
  __shared__ int s_novf;
  __shared__ unsigned int s_ovf[CS_OVF_MAX];
  if (tid == 0) s_novf = 0;
  __syncthreads();
  {
    const unsigned int *cells = P.cells + (size_t)img * P.cellWords;
    const unsigned lim = (unsigned)P.capLimit;
    // 16 independent loads per thread and round trip: the scan is one CTA per image, so it is pure latency
    for (int i0 = tid; i0 < P.cellWords; i0 += 16 * C32_THREADS) {
      unsigned v[16];
#pragma unroll
      for (int u = 0; u < 16; u++) {
        const int i = i0 + u * C32_THREADS;
        v[u] = i < P.cellWords ? __ldg(cells + i) : 0u;
      }
#pragma unroll
      for (int u = 0; u < 16; u++) {
        if (v[u] == 0) continue;
#pragma unroll
        for (int b = 0; b < 4; b++)
          if (((v[u] >> (8 * b)) & 0xff) > lim) {
            const int at = atomicAdd(&s_novf, 1);
            if (at < CS_OVF_MAX) s_ovf[at] = (unsigned)(4 * (i0 + u * C32_THREADS) + b);
          }
      }
    }
  }
  __syncthreads();
  const int novf = min(s_novf, CS_OVF_MAX);
  if (tid == 0) counters[3] = (unsigned)s_novf;          // diagnostics: cells past the limit
  if (novf == 0) return;

  __shared__ float s_v[4][C32_H][C32_VW];
  __shared__ float s_b[4][C32_H][C32_W];
  __shared__ unsigned char s_flag[30 * 8];
  __shared__ unsigned int s_drop[30 * 8];
  __shared__ int s_ndrop, s_nrm;
  __shared__ int s_rm[1024];
  SiftPoint *pts = P.pts + (size_t)img * P.ptsStride;
  if (tid == 0) s_nrm = 0;
  __syncthreads();

  for (int oi = 0; oi < novf; oi++) {
    const int cell = (int)s_ovf[oi];
    int level = 0;
    for (int l = 1; l < CS_MAX_LEVELS; l++)
      if (P.lev[l].w > 0 && cell >= P.cellBase[l]) level = l;
    const D2Level &L = P.lev[level];
    const int ci = cell - P.cellBase[level];
    const int scale = ci % CS_NUM_SCALES, blk = ci / CS_NUM_SCALES;
    const int bx = blk % P.cellsX[level], by = blk / P.cellsX[level];
    const int w = L.w, h = L.h, pitch = P.levPitch[level];
    const float *base = P.lev0Img[level] + (size_t)img * P.imgStride;
    const int cx0 = 30 * bx - 1, cy0 = 8 * by - 1;        // DoG region origin
    // vertical 9-tap of scales scale .. scale+3 (cudaSiftD.cu:1764-1772), columns cx0-4 .. cx0+35
    for (int i = tid; i < 4 * C32_H * C32_VW; i += C32_THREADS) {
      const int s = i / (C32_H * C32_VW), r = (i / C32_VW) % C32_H, c = i % C32_VW;
      const int x = min(max(cx0 - 4 + c, 0), w - 1), y = cy0 + r;
      float in[9];
#pragma unroll
      for (int j = 0; j < 9; j++) in[j] = __ldg(base + (size_t)min(max(y - 4 + j, 0), h - 1) * pitch + x);
      s_v[s][r][c] = laplace9(L.taps.k[scale + s], in[4], __fadd_rn(in[3], in[5]), __fadd_rn(in[2], in[6]),
                              __fadd_rn(in[1], in[7]), __fadd_rn(in[0], in[8]));
    }
    __syncthreads();
    // horizontal 9-tap (cudaSiftD.cu:1779-1788)
    for (int i = tid; i < 4 * C32_H * C32_W; i += C32_THREADS) {
      const int s = i / (C32_H * C32_W), r = (i / C32_W) % C32_H, c = i % C32_W;
      const float *v = &s_v[s][r][c];
      s_b[s][r][c] = laplace9(L.taps.k[scale + s], v[4], __fadd_rn(v[3], v[5]), __fadd_rn(v[2], v[6]),
                              __fadd_rn(v[1], v[7]), __fadd_rn(v[0], v[8]));
    }
    __syncthreads();
    // DoG planes scale, scale+1, scale+2 in place: plane p = blur[p+1] - blur[p] (cudaSiftD.cu:1790)
    for (int i = tid; i < C32_H * C32_W; i += C32_THREADS) {
      const int r = i / C32_W, c = i % C32_W;
      const float b0 = s_b[0][r][c], b1 = s_b[1][r][c], b2 = s_b[2][r][c], b3 = s_b[3][r][c];
      s_b[0][r][c] = __fsub_rn(b1, b0);
      s_b[1][r][c] = __fsub_rn(b2, b1);
      s_b[2][r][c] = __fsub_rn(b3, b2);
    }
    __syncthreads();
    // extrema of the cell in the reference's order: column-major, rows ascending (cudaSiftD.cu:1361-1378)
    if (tid < 240) {
      const int cxl = tid / 8, cyl = tid % 8;
      const int x = 30 * bx + cxl, y = 8 * by + cyl;
      bool ext = false;
      if (x >= 1 && x <= w - 2 && y >= 1 && y <= h - 2) {
        const float c = s_b[1][cyl + 1][cxl + 1];
        if (fabsf(c) > P.thresh) {
          bool mx = true, mn = true;
          for (int p = 0; p < 3; p++)
            for (int dy = 0; dy < 3; dy++)
              for (int dx = 0; dx < 3; dx++)
                if (p != 1 || dy != 1 || dx != 1) {
                  const float t = s_b[p][cyl + dy][cxl + dx];
                  mx = mx && (c > t); mn = mn && (c < t);
                }
          ext = c > 0.0f ? mx : mn;
        }
      }
      s_flag[tid] = ext ? 1 : 0;
    }
    __syncthreads();
    if (tid == 0) {
      int rank = 0, nd = 0;
      for (int o = 0; o < 240; o++)
        if (s_flag[o]) {
          if (rank >= P.capLimit) {
            const int x = 30 * bx + o / 8, y = 8 * by + o % 8;
            s_drop[nd++] = (unsigned)x | ((unsigned)y << 13) | ((unsigned)scale << 26) | ((unsigned)level << 29);
          }
          rank++;
        }
      s_ndrop = nd;
    }
    __syncthreads();
    // the dropped extrema that became keypoints: remember their indices
    const int count = (int)min(counters[0], (unsigned)P.maxPts);
    for (int i = tid; i < count; i += C32_THREADS) {
      const unsigned tag = __float_as_uint(pts[i].empty[0]);
      for (int d = 0; d < s_ndrop; d++)
        if (tag == s_drop[d]) {
          const int at = atomicAdd(&s_nrm, 1);
          if (at < 1024) s_rm[at] = i;
        }
    }
    __syncthreads();
  }
  // delete the remembered records: largest index first, each hole takes the then-last record
  const int nrm = min(s_nrm, 1024);
  if (nrm == 0) return;
  if (tid == 0) {
    for (int a = 1; a < nrm; a++) {                       // insertion sort, descending
      const int v = s_rm[a];
      int b = a - 1;
      while (b >= 0 && s_rm[b] < v) { s_rm[b + 1] = s_rm[b]; b--; }
      s_rm[b + 1] = v;
    }
  }
  __syncthreads();
  int count = (int)min(counters[0], (unsigned)P.maxPts);
  for (int a = 0; a < nrm; a++) {
    const int idx = s_rm[a], last = count - 1;
    if (idx != last && tid < (int)(sizeof(SiftPoint) / sizeof(float)))
      reinterpret_cast<float *>(pts + idx)[tid] = reinterpret_cast<const float *>(pts + last)[tid];
    count--;
    __syncthreads();
  }
  if (tid == 0) counters[0] = (unsigned)count;
}

int launch_cap32_fixup(const Detect2Params &p, int batch, cudaStream_t st)
{
  cap32_fixup_kernel<<<batch, C32_THREADS, 0, st>>>(p);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace cs
