// detect.cu -- fused multi-scale blur + DoG + 3x3x3 extrema + sub-pixel refinement.
//
// Behavioural spec: reference LaplaceMultiMem (cudaSiftD.cu:1753-1793, host :460-487) and
// FindPointsMultiNew (cudaSiftD.cu:1292-1431, host :489-514).  The reference writes the
// 7 DoG planes of every octave to global memory (58 MB at 1080p) and reads them back up to
// three times; here one CTA stages an input tile in shared memory, computes the 8 blurred
// scales and the 7 DoG planes of a 64x16 tile entirely on chip and tests the 62x14 interior
// for extrema, so the only global traffic is one read of the octave base image and the few
// keypoints found.  One launch covers all octaves (the tile index selects the level).
//
// All blur arithmetic works on FP32 pairs (tma.cuh: fma2 / add2, two scalar round-to-nearest
// operations on sm_90a).  A pair is (row r, row r+8) of the same column: the staged input, the vertical results and the DoG planes all live in shared memory
// as float2 {row r, row r+8}, so every 64-bit shared load is already an aligned operand pair
// and no register shuffling is needed.  Taps are duplicated (k,k) in the kernel parameters and
// consumed straight from uniform registers.
//
// Per-pixel arithmetic (which products are fused, order of the sums) is pinned to the
// reference's SASS with explicit round-to-nearest operations, so DoG values and therefore the extrema decisions
// are bit-identical to the reference's.
//
// Scheduling: persistent CTAs (4 per SM) walk the tile list; the global loads of the next tile
// are issued into registers while the current tile is still being blurred, and the slot
// allocation of a keypoint (one global atomic) is only consumed one tile later, so neither the
// DRAM latency nor the atomic round trip sits on a CTA's critical path.
//
// Deliberate difference (documented in DESIGN.md): the reference keeps at most 32
// candidates per 30x8x1 block (cudaSiftD.cu:1371,1379); no such cap exists here.
#include "common.cuh"

namespace cs {

#define DT_W 64               // DoG tile width   (62 interior columns)
#define DT_H 16               // DoG tile height  (14 interior rows)
#define DT_HP (DT_H / 2)      // row pairs (r, r+8)
#define DT_IW (DT_W + 8)      // 72 staged input columns
#define DT_PH 4               // scales blurred per phase (2 phases)
#define DT_VS 74              // float2 stride of a vertical-result row (37 16-byte chunks: odd -> the 8 row
                              // pairs of a quarter warp hit 8 different bank groups)
#define DT_THREADS 160        // CTA size
#define DT_NC 4               // DoG columns per thread in the horizontal pass (64*8/DT_NC tasks)
#define DT_VR 4               // row pairs per thread in the vertical pass (72*8/DT_VR tasks)
#define DT_MINB 4             // CTAs per SM (detect_kernel)
// shared memory, in float2 units
#define DT_SM_IN (2 * DT_HP * DT_IW)                  // staged input pairs P[j] = (in[j], in[j+8]), j = 0..15
#define DT_SM_V (DT_PH * DT_HP * DT_VS)               // vertical results of one phase
#define DT_SM_DOG ((CS_LAPLACE_S - 1) * DT_HP * DT_W) // 7 DoG planes, 16-byte chunks XOR-swizzled by the row pair
#define DT_SMEM_BYTES ((DT_SM_IN + DT_SM_V + DT_SM_DOG) * 8)   // 56832 B -> 4 CTAs per SM

// f32x2, pk/upk, fma2/mul2/add2/sub2: tma.cuh (lo = row r, hi = row r+8)

// cudaSiftD.cu:1769-1772 / 1779-1788: sum = k0*c; sum += kj*(x[-j]+x[+j]), j=1..4.
// SASS: FMUL(k1,p1); FFMA(k0,c); FFMA(k2,p2); FFMA(k3,p3); FFMA(k4,p4)  -- here on both halves at once.
__device__ __forceinline__ f32x2 lap_sym9(const float2 *k, f32x2 c, f32x2 p1, f32x2 p2, f32x2 p3, f32x2 p4)
{
  f32x2 s = mul2(pk(k[1]), p1);
  s = fma2(pk(k[0]), c, s);
  s = fma2(pk(k[2]), p2, s);
  s = fma2(pk(k[3]), p3, s);
  s = fma2(pk(k[4]), p4, s);
  return s;
}

// float index of DoG element (plane, row, col) in the swizzled pair layout
__device__ __forceinline__ int dog_index(int plane, int row, int col)
{
  const int rr = row & (DT_HP - 1);
  return (((plane * DT_HP + rr) * (DT_W / 2) + ((col >> 1) ^ rr)) << 2) + ((col & 1) << 1) + (row >> 3);
}

// ---- staging -------------------------------------------------------------------------------
// Asynchronous global->shared copies (cp.async, 4 bytes each) straight into the pair layout:
// task (g = 0..7, column c) places rows g, g+8, g+16 of the staged column as P[g] = (in[g], in[g+8])
// and P[g+8] = (in[g+8], in[g+16]).  No registers are held while the copies are in flight, so the
// next tile's loads overlap the current tile's horizontal pass and extrema test.
__device__ __forceinline__ void cp_async4(float *dst_smem, const float *src)
{
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ void tile_prefetch(float2 *s_in, const float *__restrict__ img, int w, int h,
                                              int pitch, int x0, int y0)
{
  const int tid = threadIdx.x;
  constexpr int TASKS = DT_IW * DT_HP;
  float *sf = reinterpret_cast<float *>(s_in);
  const bool interior = x0 >= 4 && x0 + DT_W + 4 <= w && y0 >= 4 && y0 + DT_H + 4 <= h;
#pragma unroll
  for (int k = 0; k < (TASKS + DT_THREADS - 1) / DT_THREADS; k++) {
    const int t = tid + k * DT_THREADS;
    if (t < TASKS) {
      const int g = t / DT_IW, cc = t - g * DT_IW;
      const float *a, *b, *c;
      if (interior) {                                   // CTA-uniform: no clamping needed
        a = img + (size_t)(y0 + g - 4) * pitch + (x0 - 4 + cc);
        b = a + (size_t)8 * pitch;
        c = b + (size_t)8 * pitch;
      } else {
        const float *col = img + min(max(x0 + cc - 4, 0), w - 1);
        a = col + (size_t)min(max(y0 + g - 4, 0), h - 1) * pitch;
        b = col + (size_t)min(max(y0 + g + 4, 0), h - 1) * pitch;
        c = col + (size_t)min(max(y0 + g + 12, 0), h - 1) * pitch;
      }
      float *d = sf + 2 * t;                            // P[g][cc]; P[g+8][cc] is DT_HP*DT_IW pairs further
      cp_async4(d, a);
      cp_async4(d + 1, b);
      cp_async4(d + 2 * DT_HP * DT_IW, b);
      cp_async4(d + 2 * DT_HP * DT_IW + 1, c);
    }
  }
  cp_async_commit();
}

// ---- blur + DoG ----------------------------------------------------------------------------
// Blur the staged tile (s_in, visible to all threads) at 8 scales and leave the 7 DoG planes in
// s_dog (pair layout, see dog_index).  (x0,y0) = image coordinates of DoG element (0,0).
// Returns this thread's candidate mask: bit d (row hr) / bit 16+d (row hr+8) is set for every
// interior pixel whose |DoG| exceeds `thresh` in one of the five testable planes, decided on the
// register copies of the DoG values -- the extrema test then only visits those pixels.
// `mid()` runs when s_in is dead (after the last vertical pass): the caller refills it there.
// Two phases of 4 scales each.  Vertical pass: task = (column, DT_VR row pairs), pair sums shared
// by the scales.  Horizontal pass + DoG: task = (row pair, DT_NC consecutive columns); the 8 lanes
// of a quarter warp take the 8 row pairs so that 128-bit shared accesses are conflict free.
template <typename Mid>
__device__ __forceinline__ unsigned int dog_tile(int w, int h, int x0, int y0, const LaplaceTaps &taps,
                                                 const float2 *s_in, float2 *s_v, float2 *s_dog,
                                                 float thresh, Mid mid)
{
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int hr = lane & 7, hg = (lane >> 3) + 4 * warp;         // horizontal task (hg < 64 / DT_NC)
  const bool hact = hg < DT_W / DT_NC;
  static_assert(4 * (DT_THREADS / 32) >= DT_W / DT_NC, "one horizontal task per thread");
  f32x2 prev[DT_NC];
  float2 amax[DT_NC];                                           // max |DoG| over planes 1..5
#pragma unroll
  for (int d = 0; d < DT_NC; d++) { prev[d] = 0ull; amax[d] = make_float2(0.0f, 0.0f); }

#pragma unroll
  for (int ph = 0; ph < CS_LAPLACE_S / DT_PH; ph++) {
    constexpr int VTASKS = DT_IW * (DT_HP / DT_VR);
#pragma unroll
    for (int vt0 = 0; vt0 < VTASKS; vt0 += DT_THREADS) {
      const int vt = vt0 + tid;
      if (vt < VTASKS) {
        const int vh = vt / DT_IW, vc = vt - vh * DT_IW;
        f32x2 in[DT_VR + 8];
#pragma unroll
        for (int i = 0; i < DT_VR + 8; i++) in[i] = pk(s_in[(DT_VR * vh + i) * DT_IW + vc]);
#pragma unroll
        for (int rr = 0; rr < DT_VR; rr++) {
          const f32x2 cc = in[rr + 4];
          const f32x2 p1 = add2(in[rr + 3], in[rr + 5]), p2 = add2(in[rr + 2], in[rr + 6]);
          const f32x2 p3 = add2(in[rr + 1], in[rr + 7]), p4 = add2(in[rr], in[rr + 8]);
#pragma unroll
          for (int s = 0; s < DT_PH; s++)
            s_v[(s * DT_HP + DT_VR * vh + rr) * DT_VS + vc] = upk(lap_sym9(taps.k[DT_PH * ph + s], cc, p1, p2, p3, p4));
        }
      }
    }
    __syncthreads();
    if (ph == CS_LAPLACE_S / DT_PH - 1) mid();
    if (hact) {
#pragma unroll
      for (int s = 0; s < DT_PH; s++) {
        const int sg = DT_PH * ph + s;
        const float4 *p = reinterpret_cast<const float4 *>(&s_v[(s * DT_HP + hr) * DT_VS + DT_NC * hg]);
        f32x2 v[DT_NC + 8];
#pragma unroll
        for (int k = 0; k < (DT_NC + 8) / 2; k++) {
          const float4 q = p[k];
          v[2 * k] = pk(make_float2(q.x, q.y));
          v[2 * k + 1] = pk(make_float2(q.z, q.w));
        }
        f32x2 o[DT_NC];
#pragma unroll
        for (int d = 0; d < DT_NC; d++)
          o[d] = lap_sym9(taps.k[sg], v[d + 4], add2(v[d + 3], v[d + 5]), add2(v[d + 2], v[d + 6]),
                          add2(v[d + 1], v[d + 7]), add2(v[d], v[d + 8]));
        if (sg > 0) {
          float4 *out = reinterpret_cast<float4 *>(s_dog) + ((sg - 1) * DT_HP + hr) * (DT_W / 2);
#pragma unroll
          for (int k = 0; k < DT_NC / 2; k++) {
            const float2 d0 = upk(sub2(o[2 * k], prev[2 * k])), d1 = upk(sub2(o[2 * k + 1], prev[2 * k + 1]));
            out[((DT_NC / 2) * hg + k) ^ hr] = make_float4(d0.x, d0.y, d1.x, d1.y);
            if (sg >= 2 && sg <= 6) {             // DoG planes 1..5 are the ones tested for extrema
              amax[2 * k].x = fmaxf(amax[2 * k].x, fabsf(d0.x)); amax[2 * k].y = fmaxf(amax[2 * k].y, fabsf(d0.y));
              amax[2 * k + 1].x = fmaxf(amax[2 * k + 1].x, fabsf(d1.x)); amax[2 * k + 1].y = fmaxf(amax[2 * k + 1].y, fabsf(d1.y));
            }
          }
        }
#pragma unroll
        for (int d = 0; d < DT_NC; d++) prev[d] = o[d];
      }
    }
    __syncthreads();
  }
  // image-border pixels can never be strict extrema in the reference (their clamped
  // neighbour is the pixel itself, cudaSiftD.cu:1308,1331-1332) -> interior only.
  unsigned int mask = 0;
  if (hact) {
#pragma unroll
    for (int d = 0; d < DT_NC; d++) {
      const int dd = DT_NC * hg + d;
      if (dd >= 1 && dd <= DT_W - 2 && x0 + dd <= w - 2) {
        if (amax[d].x > thresh) mask |= 1u << d;
        if (amax[d].y > thresh) mask |= 0x10000u << d;
      }
    }
    if (!(hr >= 1 && y0 + hr <= h - 2)) mask &= 0xffff0000u;
    if (!(hr <= DT_HP - 2 && y0 + hr + DT_HP <= h - 2)) mask &= 0x0000ffffu;
  }
  return mask;
}

// Append the pixels of a candidate mask (see dog_tile) to the tile's list as row*64+col.
__device__ __forceinline__ void list_append(unsigned int mask, unsigned short *s_list, int *s_cnt)
{
  if (mask) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int hr = lane & 7, hg = (lane >> 3) + 4 * warp;
    int at = atomicAdd(s_cnt, __popc(mask));
    while (mask) {
      const int b = __ffs(mask) - 1;
      mask &= mask - 1;
      s_list[at++] = (unsigned short)((hr + (b >> 4) * DT_HP) * DT_W + DT_NC * hg + (b & 15));
    }
  }
}

// ---- sub-pixel refinement --------------------------------------------------------------------
struct Keypoint { float x, y, scale, sharpness, edgeness, subsampling; };
#define DT_KQ 16              // keypoints a tile can park in shared memory (more: stored at once)

__device__ __forceinline__ void store_keypoint(const DetectParams &P, unsigned int idx, const Keypoint &kp)
{
  if (idx >= (unsigned)P.maxPts) idx = P.maxPts - 1;    // cudaSiftD.cu:1421
  SiftPoint *q = P.pts + idx;
  q->xpos = kp.x;
  q->ypos = kp.y;
  q->scale = kp.scale;
  q->sharpness = kp.sharpness;
  q->edgeness = kp.edgeness;
  q->subsampling = kp.subsampling;
}

// cudaSiftD.cu:1383-1429 on the shared-memory DoG planes.  pl = plane `scale` (the candidate sits in
// plane scale+1 at tile position (r, d)).  An accepted keypoint is parked in the shared queue; its
// slot in the output array is allocated (one global atomic) at the start of the next tile and the
// record written in the middle of it, so the atomic's round trip is off the critical path.
__device__ __noinline__ void refine(const float *pl, int r, int d, int gx, int gy, int scale,
                                    const DetectLevel &L, const DetectParams &P, Keypoint *s_kq, int *s_kn)
{
  float v[3][3][3];
#pragma unroll
  for (int dy = 0; dy < 3; dy++)
#pragma unroll
    for (int dx = 0; dx < 3; dx++) {
      const int o = dog_index(0, r + dy - 1, d + dx - 1);
#pragma unroll
      for (int p = 0; p < 3; p++) v[p][dy][dx] = pl[p * (DT_HP * DT_W * 2) + o];
    }
  const float val = v[1][1][1];
  float two = __fadd_rn(val, val);
  float dxx = __fsub_rn(__fsub_rn(two, v[1][1][0]), v[1][1][2]);
  float dyy = __fsub_rn(__fsub_rn(two, v[1][0][1]), v[1][2][1]);
  float dxy = __fmul_rn(0.25f, __fsub_rn(__fsub_rn(__fadd_rn(v[1][2][2], v[1][0][0]), v[1][0][2]), v[1][2][0]));
  float tra = __fadd_rn(dxx, dyy);
  float det = __fmaf_rn(dxx, dyy, -__fmul_rn(dxy, dxy));
  float tra2 = __fmul_rn(tra, tra);
  if (!(tra2 < __fmul_rn(P.edgeLimit, det))) return;
  float edge = __fdividef(tra2, det);
  float dx = __fmul_rn(0.5f, __fsub_rn(v[1][1][2], v[1][1][0]));
  float dy = __fmul_rn(0.5f, __fsub_rn(v[1][2][1], v[1][0][1]));
  float ds = __fmul_rn(0.5f, __fsub_rn(v[0][1][1], v[2][1][1]));
  float dss = __fsub_rn(__fsub_rn(two, v[2][1][1]), v[0][1][1]);
  float dxs = __fmul_rn(0.25f, __fsub_rn(__fsub_rn(__fadd_rn(v[2][1][2], v[0][1][0]), v[0][1][2]), v[2][1][0]));
  float dys = __fmul_rn(0.25f, __fsub_rn(__fsub_rn(__fadd_rn(v[2][2][1], v[0][0][1]), v[2][0][1]), v[0][2][1]));
  float idxx = __fmaf_rn(dyy, dss, -__fmul_rn(dys, dys));
  float idxy = __fmaf_rn(dys, dxs, -__fmul_rn(dxy, dss));
  float idxs = __fmaf_rn(dxy, dys, -__fmul_rn(dyy, dxs));
  float det3 = __fmaf_rn(idxs, dxs, __fmaf_rn(idxx, dxx, __fmul_rn(idxy, dxy)));
  float idet = __fdividef(1.0f, det3);
  float idyy = __fmaf_rn(dxx, dss, -__fmul_rn(dxs, dxs));
  float idys = __fmaf_rn(dxy, dxs, -__fmul_rn(dxx, dys));
  float idss = det;
  float pdx = __fmul_rn(idet, __fmaf_rn(ds, idxs, __fmaf_rn(dx, idxx, __fmul_rn(dy, idxy))));
  float pdy = __fmul_rn(idet, __fmaf_rn(ds, idys, __fmaf_rn(dy, idyy, __fmul_rn(dx, idxy))));
  float pds = __fmul_rn(idet, __fmaf_rn(idss, ds, __fmaf_rn(dx, idxs, __fmul_rn(dy, idys))));
  if (pdx < -0.5f || pdx > 0.5f || pdy < -0.5f || pdy > 0.5f || pds < -0.5f || pds > 0.5f) {
    pdx = __fdividef(dx, dxx);
    pdy = __fdividef(dy, dyy);
    pds = __fdividef(ds, dss);
  }
  float dsum = __fmaf_rn(ds, pds, __fmaf_rn(dx, pdx, __fmul_rn(dy, pdy)));
  float sc = __fmul_rn(powf(2.0f, __fdiv_rn((float)scale, (float)CS_NUM_SCALES)), exp2f(__fmul_rn(pds, P.factor)));
  if (!(sc >= L.lowestScale)) return;
  Keypoint kp;
  kp.x = __fadd_rn((float)gx, pdx);
  kp.y = __fadd_rn((float)gy, pdy);
  kp.scale = sc;
  kp.sharpness = __fmaf_rn(dsum, 0.5f, val);
  kp.edgeness = edge;
  kp.subsampling = L.subsampling;
  const int q = atomicAdd(s_kn, 1);
  if (q < DT_KQ) s_kq[q] = kp;
  else store_keypoint(P, atomicAdd(&P.counters[0], 1u), kp);
}

struct TilePos { int level, x0, y0; };
__device__ __forceinline__ TilePos decode_tile(const DetectParams &P, int t)
{
  const uint2 e = __ldg(P.tiles + t);
  TilePos tp;
  tp.level = e.x & 0xff; tp.x0 = e.x >> 8; tp.y0 = e.y;
  return tp;
}

__global__ void __launch_bounds__(DT_THREADS, DT_MINB)
detect_kernel(const __grid_constant__ DetectParams P)
{
  extern __shared__ __align__(16) float2 smem2[];
  float2 *s_v = smem2;
  float2 *s_dog = smem2 + DT_SM_V;
  float2 *s_in = s_dog + DT_SM_DOG;
  // the candidate list (at most 62*14 entries) reuses the vertical-result buffer once the blur is over
  unsigned short *s_list = reinterpret_cast<unsigned short *>(s_v);
  static_assert((DT_H - 2) * (DT_W - 2) * 2 <= DT_SM_V * 8, "candidate list fits into the vertical-result buffer");
  __shared__ int s_cnt, s_kn, s_next;
  __shared__ Keypoint s_kq[DT_KQ];
  const float thresh = P.thresh;
  const float *dogf = reinterpret_cast<const float *>(s_dog);

  int t = blockIdx.x;
  unsigned int req = 0;
  if (threadIdx.x == 0) req = gridDim.x + atomicAdd(&P.counters[2], 1u);
  TilePos tp = decode_tile(P, t);
  if (threadIdx.x == 0) { s_cnt = 0; s_kn = 0; }
  tile_prefetch(s_in, P.lev[tp.level].img, P.lev[tp.level].w, P.lev[tp.level].h, P.lev[tp.level].pitch, tp.x0, tp.y0);

  for (;;) {
    const DetectLevel &L = P.lev[tp.level];
    const int x0 = tp.x0, y0 = tp.y0;
    cp_async_wait_all();
    __syncthreads();          // staged tile visible; previous tile's extrema test and keypoint queue complete

    // keypoints parked by the previous tile: allocate their slots now, write the records in mid()
    const int nkq = min(s_kn, DT_KQ);
    unsigned int slot = 0;
    if ((int)threadIdx.x < nkq) slot = atomicAdd(&P.counters[0], 1u);

    // dynamic tile scheduler, one request ahead: publish the index requested during the previous
    // tile (the barriers of the blur make it visible before mid()), request the one after
    if (threadIdx.x == 0) {
      s_next = (int)req;
      req = gridDim.x + atomicAdd(&P.counters[2], 1u);
    }
    int tn = 0;
    bool more = false;
    TilePos tpn = tp;
    const unsigned int mask = dog_tile(L.w, L.h, x0, y0, L.taps, s_in, s_v, s_dog, thresh, [&]() {
      // the staging area is free: start the next tile's copies, retire the parked keypoints
      tn = s_next;
      more = tn < P.totalTiles;
      if (more) {
        tpn = decode_tile(P, tn);
        const DetectLevel &Ln = P.lev[tpn.level];
        tile_prefetch(s_in, Ln.img, Ln.w, Ln.h, Ln.pitch, tpn.x0, tpn.y0);
      }
      if ((int)threadIdx.x < nkq) store_keypoint(P, slot, s_kq[threadIdx.x]);
      if (threadIdx.x == 0) { s_kn = 0; s_cnt = 0; }
    });
    list_append(mask, s_list, &s_cnt);
    __syncthreads();

    // 3x3x3 extrema, only on the pixels the blur pass flagged (|DoG| > thresh at some scale); one work
    // item per (flagged pixel, scale).  Sparse tiles (the finest octave: ~2 flagged pixels per tile)
    // give a warp per item, lane j < 27 holding neighbour j of the 3x3x3 cube -- a short critical path;
    // dense tiles (coarse octaves: up to 20 % of the pixels) give a thread per item.
    const int nitems = s_cnt * CS_NUM_SCALES;
    if (nitems <= 4 * (DT_THREADS / 32)) {
      const int lane = threadIdx.x & 31;
      const int pz = lane / 9, py = (lane - 9 * pz) / 3, px = lane - 9 * pz - 3 * py;
      for (int i = threadIdx.x >> 5; i < nitems; i += DT_THREADS / 32) {
        const int ci = i / CS_NUM_SCALES, sc = i - ci * CS_NUM_SCALES;
        const int rd = s_list[ci];
        const int r = rd / DT_W, d = rd - r * DT_W;
        const float *pl = dogf + sc * (DT_HP * DT_W * 2);
        float tt = 0.0f;
        if (lane < 27) tt = pl[pz * (DT_HP * DT_W * 2) + dog_index(0, r + py - 1, d + px - 1)];
        const float c = __shfl_sync(0xffffffffu, tt, 13);          // the candidate itself: (1,1,1)
        if (!(fabsf(c) > thresh)) continue;
        const bool other = lane < 27 && lane != 13;
        const bool mx = __all_sync(0xffffffffu, !other || c > tt);
        const bool mn = __all_sync(0xffffffffu, !other || c < tt);
        if ((c > 0.0f ? mx : mn) && lane == 0) refine(pl, r, d, x0 + d, y0 + r, sc, L, P, s_kq, &s_kn);
      }
    } else {
      for (int i = threadIdx.x; i < nitems; i += DT_THREADS) {
        const int ci = i / CS_NUM_SCALES, sc = i - ci * CS_NUM_SCALES;
        const int rd = s_list[ci];
        const int r = rd / DT_W, d = rd - r * DT_W;
        const float *pl = dogf + sc * (DT_HP * DT_W * 2);
        const float c = pl[DT_HP * DT_W * 2 + dog_index(0, r, d)];
        if (!(fabsf(c) > thresh)) continue;
        bool mx = true, mn = true;
#pragma unroll
        for (int dy = 0; dy < 3; dy++)
#pragma unroll
          for (int dx = 0; dx < 3; dx++) {
            const int o = dog_index(0, r + dy - 1, d + dx - 1);
#pragma unroll
            for (int p = 0; p < 3; p++)
              if (p != 1 || dy != 1 || dx != 1) {
                const float tt = pl[p * (DT_HP * DT_W * 2) + o];
                mx = mx && (c > tt); mn = mn && (c < tt);
              }
          }
        if (c > 0.0f ? mx : mn) refine(pl, r, d, x0 + d, y0 + r, sc, L, P, s_kq, &s_kn);
      }
    }
    if (!more) break;
    t = tn; tp = tpn;
  }
  __syncthreads();
  const int nkq = min(s_kn, DT_KQ);
  if ((int)threadIdx.x < nkq) store_keypoint(P, atomicAdd(&P.counters[0], 1u), s_kq[threadIdx.x]);
}

int launch_detect(const DetectParams &p, cudaStream_t st)
{
  if (p.totalTiles <= 0) return 0;
  // per device: cudaFuncSetAttribute applies to the current device only, and SM counts may differ
  static int smsOf[64];
  int dev = 0;
  CS_CUDA(cudaGetDevice(&dev));
  dev &= 63;
  if (smsOf[dev] == 0) {
    CS_CUDA(cudaFuncSetAttribute(detect_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DT_SMEM_BYTES));
    CS_CUDA(cudaDeviceGetAttribute(&smsOf[dev], cudaDevAttrMultiProcessorCount, dev));
  }
  const int sms = smsOf[dev];
  const int grid = p.totalTiles < DT_MINB * sms ? p.totalTiles : DT_MINB * sms;
  detect_kernel<<<grid, DT_THREADS, DT_SMEM_BYTES, st>>>(p);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

// Stage-level entry point (parity tests): materialise the 7 DoG planes exactly as the
// fused detector computes them.  Plane stride = h*pitch floats (cudaSiftH.cu:184).
__global__ void __launch_bounds__(DT_THREADS)
dog_planes_kernel(const float *__restrict__ img, float *__restrict__ dog, int w, int h, int pitch,
                  int tilesX, const __grid_constant__ LaplaceTaps taps)
{
  extern __shared__ __align__(16) float2 smem2[];
  float2 *s_v = smem2;
  float2 *s_dog = smem2 + DT_SM_V;
  float2 *s_in = s_dog + DT_SM_DOG;
  const int by = blockIdx.x / tilesX, bx = blockIdx.x - by * tilesX;
  const int x0 = bx * (DT_W - 2), y0 = by * (DT_H - 2);
  tile_prefetch(s_in, img, w, h, pitch, x0, y0);
  cp_async_wait_all();
  __syncthreads();
  dog_tile(w, h, x0, y0, taps, s_in, s_v, s_dog, 0.0f, []() {});
  const float *dogf = reinterpret_cast<const float *>(s_dog);
  const size_t plane = (size_t)h * pitch;
  for (int i = threadIdx.x; i < (CS_LAPLACE_S - 1) * DT_H * DT_W; i += DT_THREADS) {
    int s = i / (DT_H * DT_W), rem = i - s * (DT_H * DT_W);
    int r = rem / DT_W, d = rem - r * DT_W;
    int gx = x0 + d, gy = y0 + r;
    if (gx < w && gy < h) dog[s * plane + (size_t)gy * pitch + gx] = dogf[dog_index(s, r, d)];
  }
}

int launch_dog_planes(const float *base, float *dog, int w, int h, int pitch, const LaplaceTaps &taps, cudaStream_t st)
{
  static bool configured[64];
  int dev = 0;
  CS_CUDA(cudaGetDevice(&dev));
  dev &= 63;
  if (!configured[dev]) {
    CS_CUDA(cudaFuncSetAttribute(dog_planes_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DT_SMEM_BYTES));
    configured[dev] = true;
  }
  int tilesX = idivup(w, DT_W - 2), tilesY = idivup(h, DT_H - 2);
  dog_planes_kernel<<<tilesX * tilesY, DT_THREADS, DT_SMEM_BYTES, st>>>(base, dog, w, h, pitch, tilesX, taps);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace cs
