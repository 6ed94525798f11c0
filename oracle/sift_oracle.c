/*
 * sift_oracle.c -- CPU restatement of the CudaSift hot path.  TEST INFRASTRUCTURE ONLY:
 * see sift_oracle.h.  Plain C, scalar, one function per reference stage; every FMA the
 * reference's SASS contains is written as an explicit fmaf() so that the
 * deterministic image stages (LowPass, ScaleDown, Laplace/DoG, extrema test) are
 * bit-identical to the reference kernels.  Build: gcc -O2 -mfma -ffp-contract=off.
 *
 * What cannot be bit-identical on a CPU (and is within ~1e-6 relative instead):
 * MUFU-based intrinsics (__fdividef, exp2f, __sinf/__cosf/__expf, rsqrtf), CUDA's
 * software powf/atan2f/expf, and the texture unit's interpolation arithmetic.
 */
#include "sift_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>

#define NUM_SCALES 5          /* cudaSiftD.h:8 */
#define LAPLACE_S  8          /* NUM_SCALES + 3, cudaSiftD.h:35 */

static inline int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }
static inline int align_up(int a, int b) { return (a % b != 0) ? (a - a % b + b) : a; }

/* ------------------------------------------------------------------ taps */

void oracle_scaledown_taps(float variance, float k[5])
{ /* cudaSiftH.cu:315-324 */
  float sum = 0.0f;
  for (int j = 0; j < 5; j++) {
    k[j] = expf((float)(-(double)(j - 2) * (j - 2) / 2.0 / variance));
    sum += k[j];
  }
  for (int j = 0; j < 5; j++) k[j] /= sum;
}

void oracle_lowpass_taps(float sigma, float k[9])
{ /* cudaSiftH.cu:408-419 */
  float sum = 0.0f;
  float ivar2 = 1.0f / (2.0f * sigma * sigma);
  for (int j = -4; j <= 4; j++) {
    k[j + 4] = expf((float)(-(double)j * j * ivar2));
    sum += k[j + 4];
  }
  for (int j = -4; j <= 4; j++) k[j + 4] /= sum;
}

void oracle_laplace_taps(int numOctaves, float initBlur, float *kernel)
{ /* cudaSiftH.cu:439-458 */
  if (numOctaves > 1) {
    float tot = sqrtf(initBlur * initBlur + 0.5f * 0.5f) / 2.0f;
    oracle_laplace_taps(numOctaves - 1, tot, kernel);
  }
  float scale = powf(2.0f, -1.0f / NUM_SCALES);
  float diffScale = powf(2.0f, 1.0f / NUM_SCALES);
  for (int i = 0; i < NUM_SCALES + 3; i++) {
    float sum = 0.0f;
    float var = scale * scale - initBlur * initBlur;
    float *k = kernel + numOctaves * 12 * 16 + 16 * i;
    for (int j = 0; j <= 4; j++) {
      k[j] = expf((float)(-(double)j * j / 2.0 / var));
      sum += (j == 0 ? 1 : 2) * k[j];
    }
    for (int j = 0; j <= 4; j++) k[j] /= sum;
    scale *= diffScale;
  }
}

/* ------------------------------------------------------------------ image stages */

/* 9-tap symmetric filter as the reference's SASS evaluates it (LowPassBlock, both
 * passes): t = rn(k3*p1); t = fma(k4,c,t); fma(k2,p2); fma(k1,p3); fma(k0,p4), where
 * k[4] is the centre tap and p_j = x[-j] + x[+j]. */
static inline float sym9_lowpass(const float k[9], float c, float p1, float p2, float p3, float p4)
{
  float t = k[3] * p1;
  t = fmaf(k[4], c, t);
  t = fmaf(k[2], p2, t);
  t = fmaf(k[1], p3, t);
  t = fmaf(k[0], p4, t);
  return t;
}

void oracle_lowpass(const float *src, float *dst, int w, int h, int pitch, float sigma)
{ /* cudaSiftD.cu:1986-2037: horizontal (shuffles) then vertical (smem ring), clamped */
  float k[9];
  oracle_lowpass_taps(sigma, k);
  float *tmp = (float *)malloc(sizeof(float) * (size_t)w * h);
  for (int y = 0; y < h; y++) {
    const float *r = src + (size_t)y * pitch;
    for (int x = 0; x < w; x++) {
#define SX(d) r[clampi(x + (d), 0, w - 1)]
      tmp[(size_t)y * w + x] = sym9_lowpass(k, SX(0), SX(1) + SX(-1), SX(2) + SX(-2),
                                            SX(3) + SX(-3), SX(4) + SX(-4));
#undef SX
    }
  }
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
#define SY(d) tmp[(size_t)clampi(y + (d), 0, h - 1) * w + x]
      dst[(size_t)y * pitch + x] = sym9_lowpass(k, SY(0), SY(-1) + SY(1), SY(-2) + SY(2),
                                                SY(-3) + SY(3), SY(-4) + SY(4));
#undef SY
    }
  free(tmp);
}

void oracle_scaledown(const float *src, float *dst, int w, int h, int pitch, int newpitch)
{ /* cudaSiftD.cu:84-168; taps variance 0.5 (cudaSiftH.cu:157) */
  float k[5];
  oracle_scaledown_taps(0.5f, k);
  int w2 = w / 2, h2 = h / 2;
  float *tmp = (float *)malloc(sizeof(float) * (size_t)w2 * h);
  for (int y = 0; y < h; y++) {
    const float *r = src + (size_t)y * pitch;
    for (int x = 0; x < w2; x++) {
#define A(j) r[clampi(2 * x + (j) - 2, 0, w - 1)]
      /* :121  k0*(a0+a4) + k1*(a1+a3) + k2*a2  ->  fma(k2,a2, fma(k0,p0, rn(k1*p1))) */
      float t = k[1] * (A(1) + A(3));
      t = fmaf(k[0], A(0) + A(4), t);
      t = fmaf(k[2], A(2), t);
      tmp[(size_t)y * w2 + x] = t;
#undef A
    }
  }
  for (int y = 0; y < h2; y++)
    for (int x = 0; x < w2; x++) {
#define R(j) tmp[(size_t)clampi(2 * y + (j) - 2, 0, h - 1) * w2 + x]
      /* :123  k2*c + k0*(r0+r4) + k1*(r1+r3)  ->  fma(k1,p1, fma(k2,c, rn(k0*p0))) */
      float t = k[0] * (R(0) + R(4));
      t = fmaf(k[2], R(2), t);
      t = fmaf(k[1], R(1) + R(3), t);
      dst[(size_t)y * newpitch + x] = t;
#undef R
    }
  free(tmp);
}

void oracle_scaleup(const float *src, float *dst, int w, int h, int pitch, int newpitch)
{ /* cudaSiftD.cu:170-190 */
  for (int yu = 0; yu < h; yu++)
    for (int xl = 0; xl < w; xl++) {
      int xr = imin(xl + 1, w - 1), yd = imin(yu + 1, h - 1);
      float vul = src[(size_t)yu * pitch + xl], vur = src[(size_t)yu * pitch + xr];
      float vdl = src[(size_t)yd * pitch + xl], vdr = src[(size_t)yd * pitch + xr];
      float *o = dst + (size_t)(2 * yu) * newpitch + 2 * xl;
      o[0] = vul;
      o[1] = 0.50f * (vul + vur);
      o[newpitch] = 0.50f * (vul + vdl);
      o[newpitch + 1] = 0.25f * (((vul + vur) + vdl) + vdr);
    }
}

/* Laplace taps k[0..4] (k[0] centre): sum = k0*c; sum += kj*(x[-j]+x[+j]) j=1..4
 * (cudaSiftD.cu:1769-1772, 1779-1788) -> SASS: t = rn(k1*p1); fma(k0,c,t); fma(k2,p2);
 * fma(k3,p3); fma(k4,p4). */
static inline float sym9_laplace(const float *k, float c, float p1, float p2, float p3, float p4)
{
  float t = k[1] * p1;
  t = fmaf(k[0], c, t);
  t = fmaf(k[2], p2, t);
  t = fmaf(k[3], p3, t);
  t = fmaf(k[4], p4, t);
  return t;
}

void oracle_dog(const float *base, float *dog, int w, int h, int pitch, const float *taps)
{ /* cudaSiftD.cu:1753-1793: vertical pass then horizontal pass, clamp to edge */
  size_t plane = (size_t)h * pitch;
  float *vert = (float *)malloc(sizeof(float) * (size_t)w * h);
  float *prev = (float *)malloc(sizeof(float) * (size_t)w * h);
  float *cur = (float *)malloc(sizeof(float) * (size_t)w * h);
  for (int s = 0; s < LAPLACE_S; s++) {
    const float *k = taps + 16 * s;
    for (int y = 0; y < h; y++)
      for (int x = 0; x < w; x++) {
#define T(d) base[(size_t)clampi(y + (d), 0, h - 1) * pitch + x]
        vert[(size_t)y * w + x] = sym9_laplace(k, T(0), T(-1) + T(1), T(-2) + T(2),
                                               T(-3) + T(3), T(-4) + T(4));
#undef T
      }
    for (int y = 0; y < h; y++) {
      const float *r = vert + (size_t)y * w;
      for (int x = 0; x < w; x++) {
#define B(d) r[clampi(x + (d), 0, w - 1)]
        cur[(size_t)y * w + x] = sym9_laplace(k, B(0), B(-1) + B(1), B(-2) + B(2),
                                              B(-3) + B(3), B(-4) + B(4));
#undef B
      }
    }
    if (s > 0)
      for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++)
          dog[(s - 1) * plane + (size_t)y * pitch + x] = cur[(size_t)y * w + x] - prev[(size_t)y * w + x];
    float *t = prev; prev = cur; cur = t;
  }
  free(vert); free(prev); free(cur);
}

/* ------------------------------------------------------------------ extrema */

/* Sub-pixel refinement + edge test of one candidate, cudaSiftD.cu:1383-1429, with the
 * FMA contraction of the reference's SASS.  Returns 1 and fills *p if the point is kept. */
static int refine_point(const float *dog, int w, int h, int pitch, int xpos, int ypos, int scale,
                        float subsampling, float lowestScale, float factor, float edgeLimit,
                        OracleSiftPoint *p)
{
  (void)w;
  const float *d1 = dog + xpos + ((size_t)ypos + (size_t)(scale + 1) * h) * pitch;
  const float *d0 = d1 - (size_t)h * pitch;   /* plane `scale`   */
  const float *d2 = d1 + (size_t)h * pitch;   /* plane `scale+2` */
  float val = d1[0];
  float two = val + val;
  float dxx = (two - d1[-1]) - d1[1];
  float dyy = (two - d1[-pitch]) - d1[pitch];
  float dxy = 0.25f * (((d1[pitch + 1] + d1[-pitch - 1]) - d1[-pitch + 1]) - d1[pitch - 1]);
  float tra = dxx + dyy;
  float det = fmaf(dxx, dyy, -(dxy * dxy));
  float tra2 = tra * tra;
  if (!(tra2 < edgeLimit * det)) return 0;
  float edge = tra2 / det;                               /* __fdividef */
  float dx = 0.5f * (d1[1] - d1[-1]);
  float dy = 0.5f * (d1[pitch] - d1[-pitch]);
  float ds = 0.5f * (d0[0] - d2[0]);
  float dss = (two - d2[0]) - d0[0];
  float dxs = 0.25f * (((d2[1] + d0[-1]) - d0[1]) - d2[-1]);
  float dys = 0.25f * (((d2[pitch] + d0[-pitch]) - d2[-pitch]) - d0[pitch]);
  float idxx = fmaf(dyy, dss, -(dys * dys));
  float idxy = fmaf(dys, dxs, -(dxy * dss));
  float idxs = fmaf(dxy, dys, -(dyy * dxs));
  float det3 = fmaf(idxs, dxs, fmaf(idxx, dxx, idxy * dxy));
  float idet = 1.0f / det3;                              /* __fdividef(1, .) */
  float idyy = fmaf(dxx, dss, -(dxs * dxs));
  float idys = fmaf(dxy, dxs, -(dxx * dys));
  float idss = det;
  float pdx = idet * fmaf(ds, idxs, fmaf(dx, idxx, dy * idxy));
  float pdy = idet * fmaf(ds, idys, fmaf(dy, idyy, dx * idxy));
  float pds = idet * fmaf(idss, ds, fmaf(dx, idxs, dy * idys));
  if (pdx < -0.5f || pdx > 0.5f || pdy < -0.5f || pdy > 0.5f || pds < -0.5f || pds > 0.5f) {
    pdx = dx / dxx;
    pdy = dy / dyy;
    pds = ds / dss;
  }
  float dsum = fmaf(ds, pds, fmaf(dx, pdx, dy * pdy));
  float sc = powf(2.0f, (float)scale / NUM_SCALES) * exp2f(pds * factor);
  if (!(sc >= lowestScale)) return 0;
  memset(p, 0, sizeof(*p));
  p->xpos = xpos + pdx;
  p->ypos = ypos + pdy;
  p->scale = sc;
  p->sharpness = fmaf(dsum, 0.5f, val);
  p->edgeness = edge;
  p->subsampling = subsampling;
  return 1;
}

/* test knobs: the reference's cap of 32 extrema per (30x8 block, scale) can be switched off, and the number of
 * extrema the cap dropped in the last oracle_extract is kept */
static int g_cap32 = 1, g_dropped = 0, g_cap_limit = 32;
void oracle_set_cap32(int on) { g_cap32 = on; }
void oracle_set_cap_limit(int n) { g_cap_limit = n > 0 ? n : 32; }   /* 32 = MEMWID, cudaSiftD.cu:1293 */
int oracle_last_dropped(void) { return g_dropped; }

int oracle_find_points(const float *dog, int w, int h, int pitch, float subsampling,
                       float lowestScale, float thresh, float factor, float edgeLimit,
                       OracleSiftPoint *pts, int *count, int maxPts, int cap32)
{ /* cudaSiftD.cu:1292-1431; block = 30 columns x 8 rows x 1 scale (cudaSiftH.cu:504-505) */
  size_t plane = (size_t)h * pitch;
  int dropped = 0;
  for (int by = 0; by * 8 < h; by++)
    for (int bx = 0; bx * 30 < w; bx++)
      for (int scale = 0; scale < NUM_SCALES; scale++) {
        int minx = bx * 30, maxx = imin(minx + 30, w);
        int yloops = imin(h - 8 * by, 8);
        int cx[240], cy[240], ncand = 0;
        /* candidates are compacted lane-major (column), then row: :1361-1376 */
        for (int x = minx; x < maxx; x++) {
          int xl = imax(x - 1, 0), xr = imin(x + 1, w - 1);
          for (int yy = 0; yy < yloops; yy++) {
            int y = 8 * by + yy;
            int yu = imax(0, y - 1), yd = imin(h - 1, y + 1);
            float d11 = dog[(scale + 1) * plane + (size_t)y * pitch + x];
            if (!(fabsf(d11) > thresh)) continue;
            float mn = INFINITY, mx = -INFINITY;
            int cols[3] = {xl, x, xr}, rows[3] = {yu, y, yd};
            for (int s = 0; s < 3; s++)
              for (int r = 0; r < 3; r++)
                for (int c = 0; c < 3; c++) {
                  if (s == 1 && r == 1 && c == 1) continue;
                  float v = dog[(scale + s) * plane + (size_t)rows[r] * pitch + cols[c]];
                  mn = fminf(mn, v);
                  mx = fmaxf(mx, v);
                }
            if ((d11 < fminf(-thresh, mn)) || (d11 > fmaxf(thresh, mx))) {
              if (cap32 && ncand >= g_cap_limit) { dropped++; continue; }   /* pos<MEMWID, tx<totbits */
              cx[ncand] = x; cy[ncand] = y; ncand++;
            }
          }
        }
        for (int i = 0; i < ncand; i++) {
          OracleSiftPoint p;
          if (refine_point(dog, w, h, pitch, cx[i], cy[i], scale, subsampling, lowestScale, factor, edgeLimit, &p)) {
            int idx = *count; (*count)++;
            if (idx >= maxPts) idx = maxPts - 1;   /* :1421 */
            pts[idx] = p;
          }
        }
      }
  return dropped;
}

/* ------------------------------------------------------------------ texture */

float oracle_tex2d(const float *img, int w, int h, int pitch, float x, float y)
{ /* CUDA linear filtering with clamp addressing and unnormalised coordinates, as measured
     on the GPU texture unit (scripts/tex_calib.py; tests/test_tex_gpu.py checks it on the H100):
       fixed-point coordinate  F = floor((x - 0.5)*256 + 0.5), texel i = F >> 8, A = F & 255
       (1.8 fixed-point weight, round to nearest); likewise B for y;
       2-D weights in 1/256 units:  w11 = (A*B + 128) >> 8, w10 = A - w11, w01 = B - w11,
       w00 = 256 - A - B + w11;  the weighted sum is formed exactly and rounded once. */
  double fx = floor(((double)x - 0.5) * 256.0 + 0.5), fy = floor(((double)y - 0.5) * 256.0 + 0.5);
  if (!(fx > -1.0e9 && fx < 1.0e9)) fx = 0.0;     /* NaN / huge coordinates */
  if (!(fy > -1.0e9 && fy < 1.0e9)) fy = 0.0;
  double ixd = floor(fx / 256.0), iyd = floor(fy / 256.0);
  int A = (int)(fx - ixd * 256.0), B = (int)(fy - iyd * 256.0);
  int i0 = (int)ixd, j0 = (int)iyd;
  int i1 = clampi(i0 + 1, 0, w - 1), j1 = clampi(j0 + 1, 0, h - 1);
  i0 = clampi(i0, 0, w - 1); j0 = clampi(j0, 0, h - 1);
  int w11 = (A * B + 128) >> 8, w10 = A - w11, w01 = B - w11, w00 = 256 - A - B + w11;
  double t00 = img[(size_t)j0 * pitch + i0], t10 = img[(size_t)j0 * pitch + i1];
  double t01 = img[(size_t)j1 * pitch + i0], t11 = img[(size_t)j1 * pitch + i1];
  return (float)((w00 * t00 + w10 * t10 + w01 * t01 + w11 * t11) * (1.0 / 256.0));
}

/* ------------------------------------------------------------------ orientation */

void oracle_orientations(const float *img, int w, int h, int pitch, OracleSiftPoint *pts,
                         int first, int last, int *count, int maxPts)
{ /* cudaSiftD.cu:972-1057 */
  first = imin(first, maxPts); last = imin(last, maxPts);
  for (int bx = first; bx < last; bx++) {
    float hist[64], gauss[11];
    float sc = pts[bx].scale;
    float i2sigma2 = -1.0f / ((4.5f * sc) * sc);           /* :982 */
    for (int t = 0; t < 11; t++) gauss[t] = expf((i2sigma2 * (t - 5)) * (t - 5));
    for (int i = 0; i < 64; i++) hist[i] = 0.0f;
    float xp = pts[bx].xpos - 4.5f, yp = pts[bx].ypos - 4.5f;
    for (int tx = 0; tx < 121; tx++) {
      int yd = tx / 11, xd = tx - yd * 11;
      float xf = xp + xd, yf = yp + yd;
      float dx = oracle_tex2d(img, w, h, pitch, xf + 1.0f, yf) - oracle_tex2d(img, w, h, pitch, xf - 1.0f, yf);
      float dy = oracle_tex2d(img, w, h, pitch, xf, yf + 1.0f) - oracle_tex2d(img, w, h, pitch, xf, yf - 1.0f);
      int bin = (int)(16.0f * atan2f(dy, dx) / 3.1416f + 16.5f);
      if (bin > 31) bin = 0;
      float grad = sqrtf(fmaf(dx, dx, dy * dy));
      hist[bin] += (grad * gauss[xd]) * gauss[yd];
    }
    for (int tx = 0; tx < 32; tx++) {                     /* :1004-1010 */
      int x1m = (tx >= 1 ? tx - 1 : tx + 31), x1p = (tx <= 30 ? tx + 1 : tx - 31);
      int x2m = (tx >= 2 ? tx - 2 : tx + 30), x2p = (tx <= 29 ? tx + 2 : tx - 30);
      hist[tx + 32] = fmaf(hist[tx], 6.0f, 4.0f * (hist[x1m] + hist[x1p])) + (hist[x2m] + hist[x2p]);
    }
    for (int tx = 0; tx < 32; tx++) {                     /* :1012-1015 */
      int x1m = (tx >= 1 ? tx - 1 : tx + 31), x1p = (tx <= 30 ? tx + 1 : tx - 31);
      float v = hist[32 + tx];
      hist[tx] = (v > hist[32 + x1m] && v >= hist[32 + x1p] ? v : 0.0f);
    }
    float maxval1 = 0.0f, maxval2 = 0.0f;
    int i1 = -1, i2 = -1;
    for (int i = 0; i < 32; i++) {                        /* :1022-1033 */
      float v = hist[i];
      if (v > maxval1) { maxval2 = maxval1; maxval1 = v; i2 = i1; i1 = i; }
      else if (v > maxval2) { maxval2 = v; i2 = i; }
    }
    float val1 = hist[32 + ((i1 + 1) & 31)], val2 = hist[32 + ((i1 + 31) & 31)];
    float peak = i1 + 0.5f * (val1 - val2) / ((2.0f * maxval1 - val1) - val2);
    pts[bx].orientation = 11.25f * (peak < 0.0f ? peak + 32.0f : peak);
    if (maxval2 > 0.8f * maxval1) {                       /* :1039-1052 */
      float v1 = hist[32 + ((i2 + 1) & 31)], v2 = hist[32 + ((i2 + 31) & 31)];
      float pk = i2 + 0.5f * (v1 - v2) / ((2.0f * maxval2 - v1) - v2);
      int idx = *count; (*count)++;
      if (idx < maxPts) {
        memset(&pts[idx], 0, sizeof(pts[idx]));
        pts[idx].xpos = pts[bx].xpos;
        pts[idx].ypos = pts[bx].ypos;
        pts[idx].scale = pts[bx].scale;
        pts[idx].sharpness = pts[bx].sharpness;
        pts[idx].edgeness = pts[bx].edgeness;
        pts[idx].orientation = 11.25f * (pk < 0.0f ? pk + 32.0f : pk);
        pts[idx].subsampling = pts[bx].subsampling;
      }
    }
  }
}

/* ------------------------------------------------------------------ descriptor */

static float fast_atan2(float y, float x)
{ /* cudaSiftD.cu:295-306 */
  float absx = fabsf(x), absy = fabsf(y);
  float a = fminf(absx, absy) / fmaxf(absx, absy);
  float s = a * a;
  float r = fmaf(s, -0.0464964749f, 0.15931422f);
  r = fmaf(s, r, -0.327622764f);
  r = s * r;
  r = fmaf(r, a, a);
  r = (absy > absx ? 1.57079637f - r : r);
  r = (x < 0 ? 3.14159274f - r : r);
  r = (y < 0 ? -r : r);
  return r;
}

static int g_q22 = 0;
int oracle_last_q22(void) { return g_q22; }   /* angi == 8 votes (quirk Q22) of the last oracle_descriptors call */

static float warp_tree_sum(float *v)
{ /* the ShiftDown reduction of cudaSiftD.cu:392-393: lane 0 of a 32-lane butterfly */
  for (int d = 16; d > 0; d /= 2)
    for (int i = 0; i < d; i++) v[i] += v[i + d];
  return v[0];
}

void oracle_descriptors(const float *img, int w, int h, int pitch, OracleSiftPoint *pts,
                        int first, int last, float subsampling)
{ /* cudaSiftD.cu:308-417 */
  float gauss[16];
  g_q22 = 0;
  for (int t = 0; t < 16; t++) {
    float d = t - 7.5f;
    gauss[t] = exp2f(((d * d) * 0.0078125f) * -1.44269502f);   /* __expf(-(t-7.5)^2/128) */
  }
  for (int bx = first; bx < last; bx++) {
    float buffer[128 + 48];
    for (int i = 0; i < 128 + 48; i++) buffer[i] = 0.0f;
    float theta = (2.0f * 3.1415f / 360.0f) * pts[bx].orientation;   /* :330 */
    float sina = sinf(theta), cosa = cosf(theta);               /* __sinf/__cosf */
    float scale = 0.75f * pts[bx].scale;
    float ssina = scale * sina, scosa = scale * cosa;
    for (int y = 0; y < 16; y++)
      for (int tx = 0; tx < 16; tx++) {
        float tt = tx - 7.5f, yy = y - 7.5f;
        /* :338-339 as contracted in SASS */
        float xpos = fmaf(-ssina, yy, tt * scosa + pts[bx].xpos) + 0.5f;
        float ypos = fmaf(scosa, yy, fmaf(tt, ssina, pts[bx].ypos)) + 0.5f;
        float dx = oracle_tex2d(img, w, h, pitch, xpos + cosa, ypos + sina) -
                   oracle_tex2d(img, w, h, pitch, xpos - cosa, ypos - sina);
        float dy = oracle_tex2d(img, w, h, pitch, xpos - sina, ypos + cosa) -
                   oracle_tex2d(img, w, h, pitch, xpos + sina, ypos - cosa);
        float grad = (gauss[y] * gauss[tx]) * sqrtf(fmaf(dx, dx, dy * dy));
        float angf = fmaf(fast_atan2(dy, dx), 4.0f / 3.1415f, 4.0f);
        int hori = (tx + 2) / 4 - 1;
        float horf = (tx - 1.5f) / 4.0f - hori, ihorf = 1.0f - horf;
        int veri = (y + 2) / 4 - 1;
        float verf = (y - 1.5f) / 4.0f - veri, iverf = 1.0f - verf;
        int angi = isnan(angf) ? 0 : (int)angf;                 /* F2I.TRUNC of NaN is 0 */
        int angp = (angi < 7 ? angi + 1 : 0);
        angf -= angi;
        float iangf = 1.0f - angf;
        int hist = 8 * (4 * veri + hori);
        int p1 = angi + hist, p2 = angp + hist;
#define VOTE(i, v) do { int ii = (i); if (ii >= 0 && ii < 128 + 48) buffer[ii] += (v); } while (0)
        if (angi == 8) g_q22 += (tx >= 2) * ((y >= 2) + (y <= 13)) + (tx <= 13) * ((y >= 2) + (y <= 13));
        if (tx >= 2) {
          float grad1 = ihorf * grad;
          if (y >= 2) { float g2 = iverf * grad1; VOTE(p1, iangf * g2); VOTE(p2, angf * g2); }
          if (y <= 13) { float g2 = verf * grad1; VOTE(p1 + 32, iangf * g2); VOTE(p2 + 32, angf * g2); }
        }
        if (tx <= 13) {
          float grad1 = horf * grad;
          if (y >= 2) { float g2 = iverf * grad1; VOTE(p1 + 8, iangf * g2); VOTE(p2 + 8, angf * g2); }
          if (y <= 13) { float g2 = verf * grad1; VOTE(p1 + 40, iangf * g2); VOTE(p2 + 40, angf * g2); }
        }
#undef VOTE
      }
    /* :391-409 normalise, clamp at 0.2, renormalise */
    float part[4], tmp[32], t1[128];
    for (int wv = 0; wv < 4; wv++) {
      for (int i = 0; i < 32; i++) tmp[i] = buffer[32 * wv + i] * buffer[32 * wv + i];
      part[wv] = warp_tree_sum(tmp);
    }
    float tsum1 = ((part[0] + part[1]) + part[2]) + part[3];
    float r1 = 1.0f / sqrtf(tsum1);                             /* rsqrtf */
    for (int i = 0; i < 128; i++) t1[i] = fminf(buffer[i] * r1, 0.2f);
    for (int wv = 0; wv < 4; wv++) {
      for (int i = 0; i < 32; i++) tmp[i] = t1[32 * wv + i] * t1[32 * wv + i];
      part[wv] = warp_tree_sum(tmp);
    }
    float tsum2 = ((part[0] + part[1]) + part[2]) + part[3];
    float r2 = 1.0f / sqrtf(tsum2);
    for (int i = 0; i < 128; i++) pts[bx].data[i] = t1[i] * r2;
    pts[bx].xpos *= subsampling;
    pts[bx].ypos *= subsampling;
    pts[bx].scale *= subsampling;
  }
}

/* ------------------------------------------------------------------ full extraction */

int oracle_extract(const float *img, int w0, int h0, int pitch0, int numOctaves,
                   float initBlur, float thresh, float lowestScale, int scaleUp,
                   OracleSiftPoint *pts, int maxPts, int *total)
{ /* cudaSiftH.cu:72-232 */
  float taps[8 * 12 * 16];
  memset(taps, 0, sizeof(taps));
  oracle_laplace_taps(numOctaves, 0.0f, taps);               /* :110 */
  int w = w0 * (scaleUp ? 2 : 1), h = h0 * (scaleUp ? 2 : 1);
  int p = align_up(w, 128);
  float *low = (float *)calloc((size_t)h * p, sizeof(float));
  float sigma = initBlur > 0.001f ? initBlur : 0.001f;       /* :112 */
  if (scaleUp) {
    float *up = (float *)calloc((size_t)h * p, sizeof(float));
    oracle_scaleup(img, up, w0, h0, pitch0, p);
    oracle_lowpass(up, low, w, h, p, sigma);
    free(up);
    lowestScale *= 2.0f;                                     /* :127 */
  } else {
    /* Q5: the reference reads the source with the destination's pitch. */
    oracle_lowpass(img, low, w, h, pitch0, sigma);
    if (pitch0 != p) { /* re-pitch so that later stages see pitch p */
      float *t = (float *)calloc((size_t)h * p, sizeof(float));
      for (int y = 0; y < h; y++) memcpy(t + (size_t)y * p, low + (size_t)y * pitch0, sizeof(float) * w);
      free(low); low = t;
    }
  }
  /* pyramid: level i has size (w>>i-ish), cudaSiftH.cu:153-159 */
  float *lev[16]; int lw[16], lh[16], lp[16];
  lev[0] = low; lw[0] = w; lh[0] = h; lp[0] = p;
  for (int i = 1; i < numOctaves; i++) {
    lw[i] = lw[i - 1] / 2; lh[i] = lh[i - 1] / 2; lp[i] = align_up(lw[i], 128);
    lev[i] = (float *)calloc((size_t)lh[i] * lp[i] + 1, sizeof(float));
    oracle_scaledown(lev[i - 1], lev[i], lw[i - 1], lh[i - 1], lp[i - 1], lp[i]);
  }
  int count = 0, numPts = 0, dropped = 0;
  for (int i = numOctaves - 1; i >= 0; i--) {                 /* coarsest octave first */
    int octave = numOctaves - i;
    float subsampling = (float)(1 << i);
    float *dog = (float *)malloc(sizeof(float) * 7 * (size_t)lh[i] * lp[i]);
    oracle_dog(lev[i], dog, lw[i], lh[i], lp[i], taps + octave * 12 * 16);
    int first = count;
    dropped += oracle_find_points(dog, lw[i], lh[i], lp[i], subsampling, lowestScale / subsampling, thresh,
                                  1.0f / NUM_SCALES, 10.0f, pts, &count, maxPts, g_cap32);
    int afterFind = count;
    if (i == 0) numPts = imin(afterFind, maxPts);              /* :115-116, quirk Q1 */
    oracle_orientations(lev[i], lw[i], lh[i], lp[i], pts, first, afterFind, &count, maxPts);
    oracle_descriptors(lev[i], lw[i], lh[i], lp[i], pts, imin(first, maxPts), imin(count, maxPts), subsampling);
    free(dog);
  }
  g_dropped = dropped;
  if (scaleUp)                                                /* :130, RescalePositions */
    for (int i = 0; i < numPts; i++) { pts[i].xpos *= 0.5f; pts[i].ypos *= 0.5f; pts[i].scale *= 0.5f; }
  for (int i = 0; i < numOctaves; i++) free(lev[i]);
  if (total) *total = imin(count, maxPts);
  return numPts;
}

/* ------------------------------------------------------------------ matcher */

static void match_rows(OracleSiftPoint *s1, int r0, int r1, const OracleSiftPoint *s2, int n2)
{ /* matching.cu:301-397.  A thread of the reference owns (row, partition) with partition
     = ((p2 mod 32) div 4); scores are a sequential k=0..127 FMA chain from 0. */
  int nblk = n2 / 32;                                        /* :325  bp2 < n2 - 31 */
  for (int r = r0; r < r1; r++) {
    const float *a = s1[r].data;
    float pmax[8], psec[8]; int pidx[8];
    for (int y = 0; y < 8; y++) { pmax[y] = 0.0f; psec[y] = 0.0f; pidx[y] = -1; }
    for (int b = 0; b < nblk; b++)
      for (int y = 0; y < 8; y++)
        for (int dy = 0; dy < 4; dy++) {
          int p2 = 32 * b + 4 * y + dy;
          const float *bb = s2[p2].data;
          float sc = 0.0f;
          for (int k = 0; k < 128; k++) sc = fmaf(a[k], bb[k], sc);
          if (sc > pmax[y]) { psec[y] = pmax[y]; pmax[y] = sc; pidx[y] = p2; }
          else if (sc > psec[y]) psec[y] = sc;
        }
    float mx = pmax[0], sec = psec[0]; int idx = pidx[0];    /* :378-390 */
    for (int y = 0; y < 8; y++)
      if (idx != pidx[y]) {
        if (pmax[y] > mx) { sec = fmaxf(mx, sec); mx = pmax[y]; idx = pidx[y]; }
        else if (pmax[y] > sec) sec = pmax[y];
      }
    s1[r].score = mx;
    s1[r].match = idx;
    s1[r].match_xpos = idx >= 0 ? s2[idx].xpos : 0.0f;       /* reference reads s2[-1] */
    s1[r].match_ypos = idx >= 0 ? s2[idx].ypos : 0.0f;
    s1[r].ambiguity = sec / (mx + 1e-6f);
  }
}

void oracle_match(OracleSiftPoint *s1, int n1, const OracleSiftPoint *s2, int n2)
{
  if (!n1 || !n2) return;                                    /* matching.cu:1095-1096 */
  match_rows(s1, 0, n1, s2, n2);
}

typedef struct { OracleSiftPoint *s1; const OracleSiftPoint *s2; int r0, r1, n2; } MatchJob;
static void *match_thread(void *arg)
{
  MatchJob *j = (MatchJob *)arg;
  match_rows(j->s1, j->r0, j->r1, j->s2, j->n2);
  return NULL;
}

void oracle_match_mt(OracleSiftPoint *s1, int n1, const OracleSiftPoint *s2, int n2, int nthreads)
{
  if (!n1 || !n2) return;
  if (nthreads < 1) nthreads = 1;
  if (nthreads > 256) nthreads = 256;
  pthread_t th[256]; MatchJob jobs[256];
  int per = (n1 + nthreads - 1) / nthreads;
  int used = 0;
  for (int t = 0; t < nthreads; t++) {
    int r0 = t * per, r1 = imin(n1, r0 + per);
    if (r0 >= r1) break;
    jobs[t].s1 = s1; jobs[t].s2 = s2; jobs[t].r0 = r0; jobs[t].r1 = r1; jobs[t].n2 = n2;
    pthread_create(&th[t], NULL, match_thread, &jobs[t]);
    used++;
  }
  for (int t = 0; t < used; t++) pthread_join(th[t], NULL);
}

/* ------------------------------------------------------------------ RANSAC homography */

static float mul_rz(float a, float b)
{ /* __fmul_rz: the double product is exact, then round toward zero */
  double p = (double)a * (double)b;
  float f = (float)p;
  if (fabs((double)f) > fabs(p)) f = nextafterf(f, 0.0f);
  return f;
}

static void invert8(float a[8][8], float inv[8][8])
{ /* matching.cu:821-905 (LU decomposition with implicit pivoting, then 8 back substitutions) */
  int indx[8], imax = 0;
  float vv[8];
  for (int i = 0; i < 8; i++) {
    float big = 0.0f;
    for (int j = 0; j < 8; j++) { float t = fabsf(a[i][j]); if (t > big) big = t; }
    vv[i] = big > 0.0f ? (float)(1.0 / (double)big) : 1e16f;
  }
  for (int j = 0; j < 8; j++) {
    for (int i = 0; i < j; i++) {
      float sum = a[i][j];
      for (int k = 0; k < i; k++) sum = fmaf(-a[i][k], a[k][j], sum);
      a[i][j] = sum;
    }
    float big = 0.0f;
    for (int i = j; i < 8; i++) {
      float sum = a[i][j];
      for (int k = 0; k < j; k++) sum = fmaf(-a[i][k], a[k][j], sum);
      a[i][j] = sum;
      float dum = vv[i] * fabsf(sum);
      if (dum >= big) { big = dum; imax = i; }
    }
    if (j != imax) {
      for (int k = 0; k < 8; k++) { float t = a[imax][k]; a[imax][k] = a[j][k]; a[j][k] = t; }
      vv[imax] = vv[j];
    }
    indx[j] = imax;
    if (a[j][j] == 0.0f) a[j][j] = 1e-16f;
    if (j != 7) {
      float dum = (float)(1.0 / (double)a[j][j]);
      for (int i = j + 1; i < 8; i++) a[i][j] *= dum;
    }
  }
  for (int j = 0; j < 8; j++) {
    float b[8];
    for (int k = 0; k < 8; k++) b[k] = 0.0f;
    b[j] = 1.0f;
    int ii = -1;
    for (int i = 0; i < 8; i++) {
      int ip = indx[i];
      float sum = b[ip];
      b[ip] = b[i];
      if (ii != -1) { for (int k = ii; k < i; k++) sum = fmaf(-a[i][k], b[k], sum); }
      else if (sum != 0.0f) ii = i;
      b[i] = sum;
    }
    for (int i = 7; i >= 0; i--) {
      float sum = b[i];
      for (int k = i + 1; k < 8; k++) sum = fmaf(-a[i][k], b[k], sum);
      b[i] = sum / a[i][i];
    }
    for (int i = 0; i < 8; i++) inv[i][j] = b[i];
  }
}

double oracle_find_homography(const OracleSiftPoint *pts, int numPts, float *homography, int *numMatches,
                              int numLoops, float minScore, float maxAmbiguity, float thresh)
{ /* matching.cu:1000-1087; samples are drawn with rand() in the reference's order */
  *numMatches = 0;
  for (int i = 0; i < 9; i++) homography[i] = (i % 4 == 0) ? 1.0f : 0.0f;
  numLoops = (numLoops + 15) / 16 * 16;
  if (numPts < 8) return 0.0;
  int *valid = (int *)malloc(sizeof(int) * numPts), numValid = 0;
  for (int i = 0; i < numPts; i++)
    if (pts[i].score > minScore && pts[i].ambiguity < maxAmbiguity) valid[numValid++] = i;
  if (numValid >= 8) {
    int *rp = (int *)malloc(sizeof(int) * 4 * (size_t)numLoops);
    for (int i = 0; i < numLoops; i++) {
      int p1 = rand() % numValid, p2 = rand() % numValid, p3 = rand() % numValid, p4 = rand() % numValid;
      while (p2 == p1) p2 = rand() % numValid;
      while (p3 == p1 || p3 == p2) p3 = rand() % numValid;
      while (p4 == p1 || p4 == p2 || p4 == p3) p4 = rand() % numValid;
      rp[4 * i] = valid[p1]; rp[4 * i + 1] = valid[p2]; rp[4 * i + 2] = valid[p3]; rp[4 * i + 3] = valid[p4];
    }
    int maxCount = -1;
    float thresh2 = thresh * thresh;
    for (int l = 0; l < numLoops; l++) {
      float a[8][8], ia[8][8], b[8], hm[8];
      for (int i = 0; i < 4; i++) {                              /* matching.cu:916-938 */
        const OracleSiftPoint *p = pts + rp[4 * l + i];
        float x1 = p->xpos, y1 = p->ypos, x2 = p->match_xpos, y2 = p->match_ypos;
        float *r1 = a[2 * i], *r2 = a[2 * i + 1];
        r1[0] = x1; r1[1] = y1; r1[2] = 1.0f; r1[3] = r1[4] = r1[5] = 0.0f; r1[6] = -x2 * x1; r1[7] = -x2 * y1;
        r2[0] = r2[1] = r2[2] = 0.0f; r2[3] = x1; r2[4] = y1; r2[5] = 1.0f; r2[6] = -y2 * x1; r2[7] = -y2 * y1;
        b[2 * i] = x2; b[2 * i + 1] = y2;
      }
      invert8(a, ia);
      for (int j = 0; j < 8; j++) {
        float sum = 0.0f;
        for (int i = 0; i < 8; i++) sum = fmaf(ia[j][i], b[i], sum);
        hm[j] = sum;
      }
      int cnt = 0;                                               /* matching.cu:969-982 */
      for (int i = 0; i < numPts; i++) {
        float x1 = pts[i].xpos, y1 = pts[i].ypos, x2 = pts[i].match_xpos, y2 = pts[i].match_ypos;
        float nomx = (mul_rz(hm[0], x1) + mul_rz(hm[1], y1)) + hm[2];
        float nomy = (mul_rz(hm[3], x1) + mul_rz(hm[4], y1)) + hm[5];
        float deno = (mul_rz(hm[6], x1) + mul_rz(hm[7], y1)) + 1.0f;
        float errx = mul_rz(x2, deno) - nomx, erry = mul_rz(y2, deno) - nomy;
        float err2 = mul_rz(errx, errx) + mul_rz(erry, erry);
        if (err2 < mul_rz(thresh2, mul_rz(deno, deno))) cnt++;
      }
      if (cnt > maxCount) { maxCount = cnt; for (int j = 0; j < 8; j++) homography[j] = hm[j]; }
    }
    *numMatches = maxCount;
    free(rp);
  }
  free(valid);
  return 0.0;
}
