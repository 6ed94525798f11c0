// sift_arith.cuh -- the reference's per-pixel arithmetic, each expression stated once.
//
// Every pyramid pixel, DoG value and refined keypoint must come out of the same rounded operations as the
// reference's.  Which products nvcc fused into FMAs, and in which order the terms are summed, was read off the
// reference's SASS; here it is pinned with explicit round-to-nearest operations (no contraction), and every kernel
// that needs one of these expressions (pyramid.cu, pyramid2.cu, detect.cu, detect2.cu, cap32.cu) calls it from here.
// A chain that some kernel runs on FP32 pairs (f32x2, tma.cuh: two pixels, each half rounded as the scalar operation)
// also has a pair form.
#pragma once

#include "tma.cuh"

namespace cs {

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }

// A tap as the operand of an FP32-pair operation: a float tap is duplicated into both halves (one register feeds both
// scalar halves), a float2 tap already is.
__device__ __forceinline__ f32x2 tap2(float k) { return pk2(k, k); }
__device__ __forceinline__ f32x2 tap2(float2 k) { return pk(k); }

// The pair forms of LowPass and ScaleDown (pa_step, pyramid2.cu) are one nested expression: the scalar form's operations
// in the evaluation order that kernel was tuned with.  The order changes only the instruction schedule, not a result.

// LowPass 9-tap (LowPassBlock, cudaSiftD.cu:2001 horizontal, :2022 / :2032 vertical), k[4] = centre tap,
// pj = x[-j] + x[+j].  SASS: FMUL(k3,p1); FFMA(k4,c); FFMA(k2,p2); FFMA(k1,p3); FFMA(k0,p4), both passes.
__device__ __forceinline__ float lowpass9(const float *k, float c, float p1, float p2, float p3, float p4)
{
  float s = __fmul_rn(k[3], p1);
  s = __fmaf_rn(k[4], c, s);
  s = __fmaf_rn(k[2], p2, s);
  s = __fmaf_rn(k[1], p3, s);
  s = __fmaf_rn(k[0], p4, s);
  return s;
}
// ... on pairs of the window x0 .. x8 (centre x4)
__device__ __forceinline__ f32x2 lowpass9(const float *k, f32x2 x0, f32x2 x1, f32x2 x2, f32x2 x3, f32x2 x4, f32x2 x5,
                                          f32x2 x6, f32x2 x7, f32x2 x8)
{
  return fma2(tap2(k[0]), add2(x0, x8),
              fma2(tap2(k[1]), add2(x1, x7),
                   fma2(tap2(k[2]), add2(x2, x6), fma2(tap2(k[4]), x4, mul2(tap2(k[3]), add2(x3, x5))))));
}

// ScaleDown horizontal 5-tap (cudaSiftD.cu:121): k0*(a0+a4) + k1*(a1+a3) + k2*a2.
// SASS: FMUL(k1,(a1+a3)); FFMA(k0,(a0+a4)); FFMA(k2,a2)
__device__ __forceinline__ float scaledown_h(const float *k, float a0, float a1, float a2, float a3, float a4)
{
  float s = __fmul_rn(k[1], __fadd_rn(a1, a3));
  s = __fmaf_rn(k[0], __fadd_rn(a0, a4), s);
  s = __fmaf_rn(k[2], a2, s);
  return s;
}

// ScaleDown vertical 5-tap (cudaSiftD.cu:123): k2*r2 + k0*(r0+r4) + k1*(r1+r3).
// SASS: FMUL(k0,(r0+r4)); FFMA(k2,r2); FFMA(k1,(r1+r3))
__device__ __forceinline__ float scaledown_v(const float *k, float r0, float r1, float r2, float r3, float r4)
{
  float s = __fmul_rn(k[0], __fadd_rn(r0, r4));
  s = __fmaf_rn(k[2], r2, s);
  s = __fmaf_rn(k[1], __fadd_rn(r1, r3), s);
  return s;
}
// ... on pairs
__device__ __forceinline__ f32x2 scaledown_v(const float *k, f32x2 r0, f32x2 r1, f32x2 r2, f32x2 r3, f32x2 r4)
{
  return fma2(tap2(k[1]), add2(r1, r3), fma2(tap2(k[2]), r2, mul2(tap2(k[0]), add2(r0, r4))));
}

// Laplace 9-tap of LaplaceMultiMem (cudaSiftD.cu:1769-1772 vertical, :1779-1788 horizontal), k[0] = centre tap,
// sum = k0*c; sum += kj*pj, j = 1..4, pj = x[-j] + x[+j] (the caller's sums: the detectors share them between
// scales).  SASS: FMUL(k1,p1); FFMA(k0,c); FFMA(k2,p2); FFMA(k3,p3); FFMA(k4,p4)
__device__ __forceinline__ float laplace9(const float *k, float c, float p1, float p2, float p3, float p4)
{
  float s = __fmul_rn(k[1], p1);
  s = __fmaf_rn(k[0], c, s);
  s = __fmaf_rn(k[2], p2, s);
  s = __fmaf_rn(k[3], p3, s);
  s = __fmaf_rn(k[4], p4, s);
  return s;
}
// ... on pairs; taps as float (k, duplicated) or float2 (k, k)
template <typename K>
__device__ __forceinline__ f32x2 laplace9(const K *k, f32x2 c, f32x2 p1, f32x2 p2, f32x2 p3, f32x2 p4)
{
  f32x2 s = mul2(tap2(k[1]), p1);
  s = fma2(tap2(k[0]), c, s);
  s = fma2(tap2(k[2]), p2, s);
  s = fma2(tap2(k[3]), p3, s);
  s = fma2(tap2(k[4]), p4, s);
  return s;
}

// Sub-pixel refinement of FindPointsMultiNew (cudaSiftD.cu:1383-1429).  v[p][dy][dx]: the 3x3x3 DoG neighbourhood,
// the extremum at [1][1][1] and at integer position (gx, gy); pow_scale() yields 2^(scale/5) of cudaSiftD.cu:1417
// (called only for extrema that pass the edge test).  Returns false when the extremum is rejected (edge test,
// cudaSiftD.cu:1390, or a scale below lowestScale, :1418); otherwise fills kp.x, y, scale, sharpness and edgeness.
// edgeLimit, factor and lowestScale are references so that a caller holding them in memory (detect.cu's refine)
// reads each one where the refinement first uses it, not before the edge test.
template <typename Pow, typename KP>
__device__ __forceinline__ bool refine_extremum(const float (&v)[3][3][3], int gx, int gy, const float &edgeLimit,
                                                const float &factor, const float &lowestScale, Pow pow_scale, KP &kp)
{
  const float val = v[1][1][1];
  float two = __fadd_rn(val, val);
  float dxx = __fsub_rn(__fsub_rn(two, v[1][1][0]), v[1][1][2]);
  float dyy = __fsub_rn(__fsub_rn(two, v[1][0][1]), v[1][2][1]);
  float dxy = __fmul_rn(0.25f, __fsub_rn(__fsub_rn(__fadd_rn(v[1][2][2], v[1][0][0]), v[1][0][2]), v[1][2][0]));
  float tra = __fadd_rn(dxx, dyy);
  float det = __fmaf_rn(dxx, dyy, -__fmul_rn(dxy, dxy));
  float tra2 = __fmul_rn(tra, tra);
  if (!(tra2 < __fmul_rn(edgeLimit, det))) return false;
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
  float sc = __fmul_rn(pow_scale(), exp2f(__fmul_rn(pds, factor)));
  if (!(sc >= lowestScale)) return false;
  kp.x = __fadd_rn((float)gx, pdx);
  kp.y = __fadd_rn((float)gy, pdy);
  kp.scale = sc;
  kp.sharpness = __fmaf_rn(dsum, 0.5f, val);
  kp.edgeness = edge;
  return true;
}

}  // namespace cs
