// pyramid2.cu -- fused, batched Gaussian pyramid: (A) LowPass + first ScaleDown in one marching kernel fed by
// TMA, (B) the remaining ScaleDowns in one launch.  Behavioural spec: reference LowPassBlock
// (cudaSiftD.cu:1986-2037, host cudaSiftH.cu:406-435) and ScaleDown (cudaSiftD.cu:84-168, host :308-338);
// per-pixel arithmetic from sift_arith.cuh (pinned to the reference's SASS), so every level is bit-identical
// to the reference's.
//
// Kernel A: a WARP owns a strip of 120 columns x R rows of the full-resolution level and marches down the rows; warps
// never talk to each other, so there is no CTA barrier anywhere.  Input rows arrive by TMA (cp.async.bulk.tensor.2d,
// 136 x 1 boxes, 8 rows in flight per warp, row index clamped by the issuing lane); each lane filters 4 columns:
// horizontal 9-tap from the staged row, vertical 9-tap over its own 9-row register window (FP32 pairs on column
// pairs), one 128-bit store of the level-0 row.  The same row is handed to the 5-tap ScaleDown through three warp
// shuffles, so level 1 is produced without re-reading level 0: HBM traffic per image = read input + write level 0
// + write level 1 (the reference: + one more read of level 0).
// Kernel B: a CTA owns an 8x8 tile of the coarsest level it produces and computes the up to three levels above it
// for that tile in shared memory (85x85 -> 41x41 -> 19x19 -> 8x8), writing the part of every level it owns: the
// four dependent launches of the reference (cudaSiftH.cu:153-157) become two.
#include "common.cuh"
#include "sift_arith.cuh"

namespace cs {

#define PA_THREADS 32      // one warp per CTA: a strip is private to its warp, so the march needs no CTA barrier
#define PA_IW CS_PA_BOX    // staged input columns x0-8 .. x0+127 (one TMA box row)
#define PA_SLOT 160        // floats between ring slots (640 B: TMA destinations are 128-byte aligned)
#define PA_NS 9            // input rows in flight per warp = depth of the register window, so ring slot = window slot

// Per-warp constants of the march ...
struct PaCtx {
  int w, h, x0, R0, R1, ia, seqEnd, Y1b, p0, p1, w1, cb, x1;
  bool own, sd;
};
// ... and what changes from step to step
struct PaRun {
  int seq;          // input row ia + seq
  int y;            // level-0 row this step produces (ia + seq - 4)
  int nextY1, trig; // next level-1 row and the level-0 row that completes it
  unsigned par;     // mbarrier phase the next wait expects (flips after slot 8: slots 0..7 then start their next use)
  float *out0;      // level-0 row y, column cb
  float *out1;      // level-1 row nextY1, column x1
};

// One marching step = input row ia+seq (row index clamped by the TMA issuer, which reproduces the reference's clamped
// row reads: cudaSiftD.cu:1997).  PH: window slot AND ring slot of this step (compile-time: the step loop is
// unrolled by 9).  The 9-row window lives in registers as two FP32 pairs per row (columns cb,cb+1 | cb+2,cb+3), so
// the vertical pass runs on pair arithmetic (tma.cuh).  EDGE: the strip touches the left or right image border (columns are
// clamped by the reading lane; the ScaleDown neighbours go through shared memory instead of shuffles).
// MAIN: the window is full -> vertical pass, level-0 store, ScaleDown.
template <int PH, bool EDGE, bool MAIN>
__device__ __forceinline__ void pa_step(const PaCtx &C, PaRun &R, f32x2 (&W)[9][2], const Taps9 &lp, const Taps5 &sdk,
                                        float *s_in, float2 *s_h2, float *s_l0, uint64_t *s_full, const CUtensorMap *map)
{
  const int lane = threadIdx.x;
  float *rowp = s_in + PH * PA_SLOT;
  mbarrier_wait(&s_full[PH], R.par);
  // ------------------------------------------------------------------ horizontal 9-tap of the input row
  float v[12];
  {
    const float4 *p = reinterpret_cast<const float4 *>(rowp + 4 * lane);       // columns cb-4 .. cb+7
    const float4 a = p[0], b = p[1], c = p[2];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    v[8] = c.x; v[9] = c.y; v[10] = c.z; v[11] = c.w;
  }
  if (EDGE) {
    if (C.cb - 4 < 0 || C.cb + 7 > C.w - 1) {                // cudaSiftD.cu:2005-2008: clamped column reads
#pragma unroll
      for (int i = 0; i < 12; i++) v[i] = rowp[clampi(C.cb - 4 + i, 0, C.w - 1) - (C.x0 - 8)];
    }
  }
  float o[4];
#pragma unroll
  for (int d = 0; d < 4; d++)
    o[d] = lowpass9(lp.k, v[d + 4], __fadd_rn(v[d + 5], v[d + 3]), __fadd_rn(v[d + 6], v[d + 2]),
                    __fadd_rn(v[d + 7], v[d + 1]), __fadd_rn(v[d + 8], v[d]));
  W[PH][0] = pk2(o[0], o[1]);
  W[PH][1] = pk2(o[2], o[3]);
  __syncwarp();                                              // every lane has consumed the slot
  if (lane == 0 && R.seq + PA_NS <= C.seqEnd) {              // refill it with the row 9 steps ahead
    mbarrier_expect_tx(&s_full[PH], PA_IW * 4);
    tma_load_2d(rowp, map, C.x0 - 8, clampi(C.ia + R.seq + PA_NS, 0, C.h - 1), &s_full[PH]);
  }
  R.seq++;
  if (!MAIN) return;
  // -------------------------------------------------------------------- vertical 9-tap -> level-0 row y
  const int y = R.y;
  float4 o4;
  {
    // window order: oldest = slot PH+1 (row y-4) ... newest = slot PH (row y+4); two columns at once
#define PAW(i, hh) W[(PH + 1 + (i)) % 9][hh]
#define PAV(hh) \
  lowpass9(lp.k, PAW(0, hh), PAW(1, hh), PAW(2, hh), PAW(3, hh), PAW(4, hh), PAW(5, hh), PAW(6, hh), PAW(7, hh), PAW(8, hh))
    const float2 lo = upk(PAV(0)), hi = upk(PAV(1));
#undef PAV
#undef PAW
    o4 = make_float4(lo.x, lo.y, hi.x, hi.y);
  }
  if (C.own && y >= C.R0 && y < C.R1) {
    if (!EDGE || C.cb + 3 < C.w) *reinterpret_cast<float4 *>(R.out0) = o4;
    else {
      if (C.cb < C.w) R.out0[0] = o4.x;
      if (C.cb + 1 < C.w) R.out0[1] = o4.y;
      if (C.cb + 2 < C.w) R.out0[2] = o4.z;
    }
  }
  R.out0 += C.p0;
  R.y = y + 1;
  if (!C.sd) return;
  // -------------------------------------------------------------------- ScaleDown: horizontal 5-tap of row y
  float a[7];                                                // columns cb-2 .. cb+4
  if (!EDGE) {
    a[0] = __shfl_up_sync(0xffffffffu, o4.z, 1);
    a[1] = __shfl_up_sync(0xffffffffu, o4.w, 1);
    a[2] = o4.x; a[3] = o4.y; a[4] = o4.z; a[5] = o4.w;
    a[6] = __shfl_down_sync(0xffffffffu, o4.x, 1);
  } else {
    __syncwarp();                                            // the previous row's reads are done
    *reinterpret_cast<float4 *>(s_l0 + 4 * lane) = o4;       // s_l0[i] = column x0-4+i
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 7; i++) a[i] = s_l0[clampi(clampi(C.cb - 2 + i, 0, C.w - 1) - (C.x0 - 4), 0, 4 * PA_THREADS - 1)];
  }
  float2 *h2 = s_h2 + lane;                                  // [row & 7][lane] and again at [8 + (row & 7)][lane]: a private
  {                                                          // column, stored twice so that any 5 consecutive rows are contiguous
    const float2 hv = make_float2(scaledown_h(sdk.k, a[0], a[1], a[2], a[3], a[4]),
                                  scaledown_h(sdk.k, a[2], a[3], a[4], a[5], a[6]));
    float2 *hw = h2 + (y & 7) * PA_THREADS;
    hw[0] = hv;
    hw[8 * PA_THREADS] = hv;
  }
  // ---------------------------------------------------------------------- ... vertical 5-tap -> the level-1 row that is complete
  if (R.nextY1 < C.Y1b && R.trig <= y) {
    f32x2 q[5];
    if (y >= 4 && R.trig == 2 * R.nextY1 + 2) {             // rows y-4 .. y, no clamping (y-4 = y+4 mod 8)
#pragma unroll
      for (int j = 0; j < 5; j++) q[j] = pk(h2[(((y + 4) & 7) + j) * PA_THREADS]);
    } else {
#pragma unroll
      for (int j = 0; j < 5; j++) q[j] = pk(h2[(clampi(2 * R.nextY1 - 2 + j, 0, C.h - 1) & 7) * PA_THREADS]);
    }
    const f32x2 s = scaledown_v(sdk.k, q[0], q[1], q[2], q[3], q[4]);     // both columns at once
    if (C.own) {
      const float2 r = upk(s);
      if (!EDGE || C.x1 + 1 < C.w1) *reinterpret_cast<float2 *>(R.out1) = r;
      else if (C.x1 < C.w1) R.out1[0] = r.x;
    }
    R.out1 += C.p1;
    R.nextY1++;
    R.trig = min(2 * R.nextY1 + 2, C.h - 1);
  }
}

template <bool EDGE>
__device__ __forceinline__ void pa_march(const PaCtx &C, PaRun &R, const Taps9 &lp, const Taps5 &sdk, float *s_in, float2 *s_h2,
                                         float *s_l0, uint64_t *s_full, const CUtensorMap *map)
{
  f32x2 W[9][2];
  // the first 8 rows only fill the window (seqEnd >= 8 always)
#define PA_PRO(p) pa_step<(p), EDGE, false>(C, R, W, lp, sdk, s_in, s_h2, s_l0, s_full, map);
  PA_PRO(0) PA_PRO(1) PA_PRO(2) PA_PRO(3) PA_PRO(4) PA_PRO(5) PA_PRO(6) PA_PRO(7)
#undef PA_PRO
#define PA_STEP(p) { if (R.seq > C.seqEnd) break; pa_step<(p), EDGE, true>(C, R, W, lp, sdk, s_in, s_h2, s_l0, s_full, map); }
  for (;;) {
    PA_STEP(8)
    R.par ^= 1u;                                             // slots 0..7 start their next use
    PA_STEP(0) PA_STEP(1) PA_STEP(2) PA_STEP(3) PA_STEP(4) PA_STEP(5) PA_STEP(6) PA_STEP(7)
  }
#undef PA_STEP
}

#ifndef PA_MINB
#define PA_MINB 1
#endif
__global__ void __launch_bounds__(PA_THREADS, PA_MINB)
pyr_lowpass_sd_kernel(const __grid_constant__ PyrAParams P)
{
  __shared__ __align__(128) float s_in[PA_NS * PA_SLOT];
  __shared__ __align__(16) float s_l0[4 * PA_THREADS];         // level-0 row of an edge strip (ScaleDown neighbours)
  __shared__ __align__(8) float2 s_h2[16 * PA_THREADS];        // [row & 7][lane] (+ a second copy 8 rows further): private columns
  __shared__ __align__(8) uint64_t s_full[PA_NS];

  const int lane = threadIdx.x;
  const int strip = blockIdx.x % P.stripsX, rb = blockIdx.x / P.stripsX, img = blockIdx.y;
  PaCtx C;
  C.w = P.w; C.h = P.h;
  C.x0 = strip * CS_PA_OWN;
  C.R0 = rb * P.rowsPerCta;
  C.R1 = (rb == P.rowBlocks - 1) ? C.h : min(C.R0 + P.rowsPerCta, C.h);
  C.sd = P.lev1 != nullptr;
  const int Y1a = C.R0 >> 1;
  C.Y1b = C.sd ? ((rb == P.rowBlocks - 1) ? P.h1 : min(C.R1 >> 1, P.h1)) : 0;
  // level-0 rows this warp computes: its own rows plus what its level-1 rows need
  const int ya = C.sd ? max(C.R0 - 2, 0) : C.R0;
  const int yb = C.sd ? min(max(C.R1 - 1, 2 * C.Y1b), C.h - 1) : C.R1 - 1;
  C.ia = ya - 4;                                              // input rows ia .. yb+4 (clamped when loaded)
  C.seqEnd = yb + 4 - C.ia;
  C.p0 = P.p0; C.p1 = P.p1; C.w1 = P.w1;
  const CUtensorMap *map = P.inMaps + img;
  C.cb = C.x0 - 4 + 4 * lane;                                 // level-0 columns cb .. cb+3
  C.own = lane >= 1 && lane <= 30;                            // owned columns x0 .. x0+119
  C.x1 = (C.x0 >> 1) + 2 * (lane - 1);                        // this lane's two level-1 columns
  PaRun R;
  R.seq = 0; R.y = ya; R.par = 0;
  R.nextY1 = Y1a; R.trig = min(2 * Y1a + 2, C.h - 1);
  R.out0 = P.lev0 + (size_t)img * P.lev0Stride + (ptrdiff_t)ya * C.p0 + C.cb;
  R.out1 = C.sd ? P.lev1 + (size_t)img * P.lev1Stride + (ptrdiff_t)Y1a * C.p1 + C.x1 : nullptr;

  if (lane == 0) {
    for (int i = 0; i < PA_NS; i++) mbarrier_init(&s_full[i], 1);
    mbarrier_init_fence();
    for (int i = 0; i < PA_NS; i++) {                         // the maps are kernel parameters: no descriptor fence needed
      mbarrier_expect_tx(&s_full[i], PA_IW * 4);
      tma_load_2d(s_in + i * PA_SLOT, map, C.x0 - 8, clampi(C.ia + i, 0, C.h - 1), &s_full[i]);
    }
  }
  __syncwarp();
  const Taps9 lp = P.lp;
  const Taps5 sdk = P.sd;
  const bool edge = (C.x0 == 0) || (C.x0 + PA_IW - 8 > C.w);   // some staged column lies outside the image
  if (edge) pa_march<true>(C, R, lp, sdk, s_in, s_h2, s_l0, s_full, map);
  else pa_march<false>(C, R, lp, sdk, s_in, s_h2, s_l0, s_full, map);
}

const void *pyr_a_func() { return (const void *)pyr_lowpass_sd_kernel; }

int launch_pyr_a(const PyrAParams &p, int batch, cudaStream_t st)
{
  dim3 grid(p.stripsX * p.rowBlocks, batch);
  pyr_lowpass_sd_kernel<<<grid, PA_THREADS, 0, st>>>(p);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------
// Kernel B: a chain of up to 3 ScaleDowns for one 8x8 tile of the last level.
// ---------------------------------------------------------------------------------------
#define PB_THREADS 256
#define PB_T 8
#define PB_N1 (2 * PB_T + 3)      // 19
#define PB_N2 (2 * PB_N1 + 3)     // 41
#define PB_N3 (2 * PB_N2 + 3)     // 85

// One ScaleDown inside shared memory.  src: NIN x NIN region of a level whose element (0,0) is pixel (sx0, sy0);
// dst: NOUT x NOUT region of the next level with origin (dx0, dy0) = ((sx0+2)/2, (sy0+2)/2), NIN = 2 NOUT + 3.
// CLAMP: coordinates are clamped to the image first (cudaSiftD.cu:98-99,113), then to the region; tiles whose
// regions lie inside the images on every level take the CLAMP = false path (plain strided reads).
template <int NOUT, bool CLAMP>
__device__ __forceinline__ void pb_scaledown(const float *src, int sx0, int sy0, int sw, int sh, float *tmp, float *dst,
                                             int dx0, int dy0, const Taps5 &k)
{
  constexpr int NIN = 2 * NOUT + 3;
  for (int i = threadIdx.x; i < NIN * NOUT; i += PB_THREADS) {      // horizontal: rows of src x columns of dst
    const int r = i / NOUT, c = i - r * NOUT;
    const float *row = src + r * NIN;
    float a[5];
    if (CLAMP) {
#pragma unroll
      for (int j = 0; j < 5; j++) a[j] = row[clampi(clampi(2 * (dx0 + c) - 2 + j, 0, sw - 1) - sx0, 0, NIN - 1)];
    } else {
#pragma unroll
      for (int j = 0; j < 5; j++) a[j] = row[2 * c + j];
    }
    tmp[i] = scaledown_h(k.k, a[0], a[1], a[2], a[3], a[4]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NOUT * NOUT; i += PB_THREADS) {
    const int r = i / NOUT, c = i - r * NOUT;
    float q[5];
    if (CLAMP) {
#pragma unroll
      for (int j = 0; j < 5; j++) q[j] = tmp[clampi(clampi(2 * (dy0 + r) - 2 + j, 0, sh - 1) - sy0, 0, NIN - 1) * NOUT + c];
    } else {
#pragma unroll
      for (int j = 0; j < 5; j++) q[j] = tmp[(2 * r + j) * NOUT + c];
    }
    dst[i] = scaledown_v(k.k, q[0], q[1], q[2], q[3], q[4]);
  }
  __syncthreads();
}

// write the part of an N x N region (origin rx0, ry0) that this tile owns: pixels [ox, ox+ON) x [oy, oy+ON)
template <int N, int ON>
__device__ __forceinline__ void pb_store(const float *reg, int rx0, int ry0, float *img, int w, int h, int pitch, int ox, int oy)
{
  for (int i = threadIdx.x; i < ON * ON; i += PB_THREADS) {
    const int r = i / ON, c = i - r * ON;
    const int gx = ox + c, gy = oy + r;
    if (gx < w && gy < h) img[(size_t)gy * pitch + gx] = reg[(gy - ry0) * N + (gx - rx0)];
  }
}

// chain of STEPS ScaleDowns for the 8x8 tile (bx, by) of the last level
template <int STEPS, bool CLAMP>
__device__ __forceinline__ void pb_chain(const PyrBParams &P, int img, float *bufA, float *bufT, float *bufB)
{
  constexpr int N0 = PB_T, N1 = 2 * N0 + 3, N2 = 2 * N1 + 3, N3 = 2 * N2 + 3;
  constexpr int NS = STEPS == 3 ? N3 : (STEPS == 2 ? N2 : N1);          // source region
  int ox[4], oy[4];
  ox[0] = blockIdx.x * PB_T; oy[0] = blockIdx.y * PB_T;
#pragma unroll
  for (int k = 1; k <= 3; k++) { ox[k] = 2 * ox[k - 1] - 2; oy[k] = 2 * oy[k - 1] - 2; }
  {
    const float *src = P.img[0] + (size_t)img * P.stride[0];
    const int sx0 = ox[STEPS], sy0 = oy[STEPS];
    for (int i = threadIdx.x; i < NS * NS; i += PB_THREADS) {
      const int r = i / NS, c = i - r * NS;
      if (CLAMP) bufA[i] = __ldg(src + (size_t)clampi(sy0 + r, 0, P.h[0] - 1) * P.pitch[0] + clampi(sx0 + c, 0, P.w[0] - 1));
      else bufA[i] = __ldg(src + (size_t)(sy0 + r) * P.pitch[0] + sx0 + c);
    }
  }
  __syncthreads();
  // level s is produced from region index STEPS-s+1 into region index STEPS-s
  if (STEPS == 3) {
    pb_scaledown<N2, CLAMP>(bufA, ox[3], oy[3], P.w[0], P.h[0], bufT, bufB, ox[2], oy[2], P.sd);
    pb_store<N2, 4 * PB_T>(bufB, ox[2], oy[2], P.img[1] + (size_t)img * P.stride[1], P.w[1], P.h[1], P.pitch[1], 4 * ox[0], 4 * oy[0]);
    pb_scaledown<N1, CLAMP>(bufB, ox[2], oy[2], P.w[1], P.h[1], bufT, bufA, ox[1], oy[1], P.sd);
    pb_store<N1, 2 * PB_T>(bufA, ox[1], oy[1], P.img[2] + (size_t)img * P.stride[2], P.w[2], P.h[2], P.pitch[2], 2 * ox[0], 2 * oy[0]);
    pb_scaledown<N0, CLAMP>(bufA, ox[1], oy[1], P.w[2], P.h[2], bufT, bufB, ox[0], oy[0], P.sd);
    pb_store<N0, PB_T>(bufB, ox[0], oy[0], P.img[3] + (size_t)img * P.stride[3], P.w[3], P.h[3], P.pitch[3], ox[0], oy[0]);
  } else if (STEPS == 2) {
    pb_scaledown<N1, CLAMP>(bufA, ox[2], oy[2], P.w[0], P.h[0], bufT, bufB, ox[1], oy[1], P.sd);
    pb_store<N1, 2 * PB_T>(bufB, ox[1], oy[1], P.img[1] + (size_t)img * P.stride[1], P.w[1], P.h[1], P.pitch[1], 2 * ox[0], 2 * oy[0]);
    pb_scaledown<N0, CLAMP>(bufB, ox[1], oy[1], P.w[1], P.h[1], bufT, bufA, ox[0], oy[0], P.sd);
    pb_store<N0, PB_T>(bufA, ox[0], oy[0], P.img[2] + (size_t)img * P.stride[2], P.w[2], P.h[2], P.pitch[2], ox[0], oy[0]);
  } else {
    pb_scaledown<N0, CLAMP>(bufA, ox[1], oy[1], P.w[0], P.h[0], bufT, bufB, ox[0], oy[0], P.sd);
    pb_store<N0, PB_T>(bufB, ox[0], oy[0], P.img[1] + (size_t)img * P.stride[1], P.w[1], P.h[1], P.pitch[1], ox[0], oy[0]);
  }
}

__global__ void __launch_bounds__(PB_THREADS)
pyr_chain_kernel(const __grid_constant__ PyrBParams P)
{
  extern __shared__ __align__(16) float pb_smem[];
  float *bufA = pb_smem;                       // up to 85 x 85
  float *bufT = bufA + PB_N3 * PB_N3;          // horizontal results, up to 85 x 41
  float *bufB = bufT + PB_N3 * PB_N2;          // up to 41 x 41
  const int img = blockIdx.z;
  // the tile needs no clamping if its region lies inside the image on every level it reads
  bool inside = true;
  {
    int x = blockIdx.x * PB_T, y = blockIdx.y * PB_T, n = PB_T;
    for (int s = P.steps; s >= 0; s--) {       // s = level index in P (steps = last level)
      if (x < 0 || y < 0 || x + n > P.w[s] || y + n > P.h[s]) inside = false;
      x = 2 * x - 2; y = 2 * y - 2; n = 2 * n + 3;
    }
  }
  if (P.steps == 3) { if (inside) pb_chain<3, false>(P, img, bufA, bufT, bufB); else pb_chain<3, true>(P, img, bufA, bufT, bufB); }
  else if (P.steps == 2) { if (inside) pb_chain<2, false>(P, img, bufA, bufT, bufB); else pb_chain<2, true>(P, img, bufA, bufT, bufB); }
  else { if (inside) pb_chain<1, false>(P, img, bufA, bufT, bufB); else pb_chain<1, true>(P, img, bufA, bufT, bufB); }
}

static int g_pb_configured[64];
#define PB_SMEM_BYTES ((PB_N3 * PB_N3 + PB_N3 * PB_N2 + PB_N2 * PB_N2) * 4)

int launch_pyr_b(const PyrBParams &p, int batch, cudaStream_t st)
{
  if (p.steps < 1) return 0;
  int dev = 0;
  CS_CUDA(cudaGetDevice(&dev));
  if (dev < 64 && !g_pb_configured[dev]) {
    CS_CUDA(cudaFuncSetAttribute(pyr_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PB_SMEM_BYTES));
    g_pb_configured[dev] = 1;
  }
  // tiles must cover every level of the chain (integer halving can leave a level wider than twice the next)
  int tx = 1, ty = 1;
  for (int s = 1; s <= p.steps; s++) {
    const int on = PB_T << (p.steps - s);
    tx = tx > idivup(p.w[s], on) ? tx : idivup(p.w[s], on);
    ty = ty > idivup(p.h[s], on) ? ty : idivup(p.h[s], on);
  }
  dim3 grid(tx, ty, batch);
  pyr_chain_kernel<<<grid, PB_THREADS, PB_SMEM_BYTES, st>>>(p);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace cs
