// pyramid.cu -- Gaussian pyramid stages: LowPass, ScaleDown, ScaleUp.
//
// Behavioural spec: reference cudaSiftD.cu:1986-2037 (LowPassBlock), :84-168 (ScaleDown),
// :170-190 (ScaleUp) and their host launchers cudaSiftH.cu:308-351, 406-435.
// These are new kernels (shared-memory tiles, 128-bit shared/global accesses); what is
// kept from the reference is the arithmetic of every output pixel (sift_arith.cuh), so
// that the pyramid is bit-identical to the reference's (and to oracle/sift_oracle.c).
#include "common.cuh"
#include "sift_arith.cuh"

namespace cs {

// ---------------------------------------------------------------------------------------
// LowPass: 9-tap separable Gaussian, horizontal then vertical, clamp-to-edge.
// Tile: 128 x 32 outputs per CTA, 256 threads.
// ---------------------------------------------------------------------------------------
#define LP_W 128
#define LP_H 32
#define LP_R 4
#define LP_IW (LP_W + 2 * LP_R)   // 136
#define LP_IH (LP_H + 2 * LP_R)   // 40

__global__ void __launch_bounds__(256, 4)      // 510 CTAs at 1080p fit one wave (132 x 4)
lowpass_kernel(const float *__restrict__ src, int srcPitch, float *__restrict__ dst, int dstPitch,
               int w, int h, const __grid_constant__ Taps9 taps)
{
  __shared__ __align__(16) float s_in[LP_IH][LP_IW];
  __shared__ __align__(16) float s_h[LP_IH][LP_W];
  const int tid = threadIdx.x;
  const int x0 = blockIdx.x * LP_W, y0 = blockIdx.y * LP_H;

  // stage the input tile (+halo), clamped.  All loads of a thread are issued before the
  // first shared-memory store so that their DRAM latencies overlap (one round trip).
  const bool interior = (x0 >= LP_R) && (x0 + LP_W + LP_R <= w) && ((srcPitch & 3) == 0) &&
                        ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
  if (interior) {
    // 40 rows x 34 float4 (the row segment starts at x0-4, a multiple of 4 floats)
    constexpr int V4 = LP_IW / 4, N = (LP_IH * V4 + 255) / 256;
    float4 v[N];
#pragma unroll
    for (int k = 0; k < N; k++) {
      int i = tid + 256 * k;
      int r = i / V4, c = i - r * V4;
      int gy = clampi(y0 + r - LP_R, 0, h - 1);
      v[k] = (i < LP_IH * V4) ? __ldg(reinterpret_cast<const float4 *>(src + (size_t)gy * srcPitch + x0 - LP_R) + c)
                              : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int k = 0; k < N; k++) {
      int i = tid + 256 * k;
      if (i < LP_IH * V4) reinterpret_cast<float4 *>(&s_in[0][0])[i] = v[k];
    }
  } else {
    constexpr int N = (LP_IH * LP_IW + 255) / 256;
    float v[N];
#pragma unroll
    for (int k = 0; k < N; k++) {
      int i = tid + 256 * k;
      int r = i / LP_IW, c = i - r * LP_IW;
      int gy = clampi(y0 + r - LP_R, 0, h - 1), gx = clampi(x0 + c - LP_R, 0, w - 1);
      v[k] = (i < LP_IH * LP_IW) ? __ldg(src + (size_t)gy * srcPitch + gx) : 0.0f;
    }
#pragma unroll
    for (int k = 0; k < N; k++) {
      int i = tid + 256 * k;
      if (i < LP_IH * LP_IW) (&s_in[0][0])[i] = v[k];
    }
  }
  __syncthreads();

  // horizontal pass: task = (row, 4 consecutive columns)
  for (int t = tid; t < LP_IH * (LP_W / 4); t += 256) {
    int r = t / (LP_W / 4), seg = t - r * (LP_W / 4);
    const float4 *p = reinterpret_cast<const float4 *>(&s_in[r][4 * seg]);
    float4 a = p[0], b = p[1], c = p[2];
    float v[12] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y, c.z, c.w};
    float o[4];
#pragma unroll
    for (int d = 0; d < 4; d++)
      o[d] = lowpass9(taps.k, v[d + 4], __fadd_rn(v[d + 5], v[d + 3]), __fadd_rn(v[d + 6], v[d + 2]),
                      __fadd_rn(v[d + 7], v[d + 1]), __fadd_rn(v[d + 8], v[d]));
    *reinterpret_cast<float4 *>(&s_h[r][4 * seg]) = make_float4(o[0], o[1], o[2], o[3]);
  }
  __syncthreads();

  // vertical pass: thread = (4 columns, 4 rows)
  {
    const int cg = tid & 31, rg = tid >> 5;
    float4 v[12];
#pragma unroll
    for (int i = 0; i < 12; i++) v[i] = *reinterpret_cast<const float4 *>(&s_h[4 * rg + i][4 * cg]);
    const int gx = x0 + 4 * cg;
#pragma unroll
    for (int d = 0; d < 4; d++) {
      const int gy = y0 + 4 * rg + d;
      float4 o;
#define LPV(f)                                                                                      \
  lowpass9(taps.k, v[d + 4].f, __fadd_rn(v[d + 3].f, v[d + 5].f), __fadd_rn(v[d + 2].f, v[d + 6].f), \
           __fadd_rn(v[d + 1].f, v[d + 7].f), __fadd_rn(v[d].f, v[d + 8].f))
      o.x = LPV(x); o.y = LPV(y); o.z = LPV(z); o.w = LPV(w);
#undef LPV
      if (gy < h) {
        float *out = dst + (size_t)gy * dstPitch + gx;
        if (gx + 3 < w && ((dstPitch & 3) == 0)) {
          *reinterpret_cast<float4 *>(out) = o;
        } else {
          if (gx < w) out[0] = o.x;
          if (gx + 1 < w) out[1] = o.y;
          if (gx + 2 < w) out[2] = o.z;
          if (gx + 3 < w) out[3] = o.w;
        }
      }
    }
  }
}

int launch_lowpass(const float *src, int srcPitch, float *dst, int dstPitch, int w, int h,
                   const Taps9 &taps, cudaStream_t st)
{
  dim3 grid(idivup(w, LP_W), idivup(h, LP_H));
  lowpass_kernel<<<grid, 256, 0, st>>>(src, srcPitch, dst, dstPitch, w, h, taps);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------
// ScaleDown: 5-tap separable Gaussian (variance 0.5) fused with 2x decimation.
// Tile: 64 x 16 outputs per CTA, 256 threads.  out(x',y') = sum k_i k_j in(2x'+i, 2y'+j).
// ---------------------------------------------------------------------------------------
#define SD_W 64
#define SD_H 16
#define SD_IW (2 * SD_W + 4)   // 132
#define SD_IH (2 * SD_H + 3)   // 35

__global__ void __launch_bounds__(256)
scaledown_kernel(const float *__restrict__ src, float *__restrict__ dst, int w, int h, int pitch,
                 int newpitch, const __grid_constant__ Taps5 taps, long long srcStride, long long dstStride)
{
  src += (size_t)blockIdx.z * srcStride;      // batched launch: image blockIdx.z
  dst += (size_t)blockIdx.z * dstStride;
  __shared__ __align__(16) float s_in[SD_IH][SD_IW];
  __shared__ __align__(16) float s_h[SD_IH][SD_W];
  const int tid = threadIdx.x;
  const int ox0 = blockIdx.x * SD_W, oy0 = blockIdx.y * SD_H;   // output-space origin
  const int w2 = w / 2, h2 = h / 2;

  {
    constexpr int N = (SD_IH * SD_IW + 255) / 256;
    float v[N];
#pragma unroll
    for (int k = 0; k < N; k++) {       // all loads first: one DRAM round trip per thread
      int i = tid + 256 * k;
      int r = i / SD_IW, c = i - r * SD_IW;
      int gy = clampi(2 * oy0 + r - 2, 0, h - 1), gx = clampi(2 * ox0 + c - 2, 0, w - 1);
      v[k] = (i < SD_IH * SD_IW) ? __ldg(src + (size_t)gy * pitch + gx) : 0.0f;
    }
#pragma unroll
    for (int k = 0; k < N; k++) {
      int i = tid + 256 * k;
      if (i < SD_IH * SD_IW) (&s_in[0][0])[i] = v[k];
    }
  }
  __syncthreads();

  // horizontal 5-tap
  for (int t = tid; t < SD_IH * SD_W; t += 256) {
    int r = t / SD_W, x = t - r * SD_W;
    const float2 *p = reinterpret_cast<const float2 *>(&s_in[r][2 * x]);
    float2 a01 = p[0], a23 = p[1], a45 = p[2];
    s_h[r][x] = scaledown_h(taps.k, a01.x, a01.y, a23.x, a23.y, a45.x);
  }
  __syncthreads();

  // vertical 5-tap
  for (int t = tid; t < SD_H * SD_W; t += 256) {
    int y = t / SD_W, x = t - y * SD_W;
    int gx = ox0 + x, gy = oy0 + y;
    if (gx < w2 && gy < h2) {
      dst[(size_t)gy * newpitch + gx] =
          scaledown_v(taps.k, s_h[2 * y][x], s_h[2 * y + 1][x], s_h[2 * y + 2][x], s_h[2 * y + 3][x], s_h[2 * y + 4][x]);
    }
  }
}

int launch_scaledown(const float *src, float *dst, int w, int h, int pitch, int newpitch,
                     const Taps5 &taps, cudaStream_t st, int batch, long long srcStride, long long dstStride)
{
  if (w / 2 < 1 || h / 2 < 1) return 0;
  dim3 grid(idivup(w / 2, SD_W), idivup(h / 2, SD_H), batch);
  scaledown_kernel<<<grid, 256, 0, st>>>(src, dst, w, h, pitch, newpitch, taps, srcStride, dstStride);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------
// ScaleUp: 2x bilinear upsample (cudaSiftD.cu:170-190).  One thread per source pixel.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
scaleup_kernel(const float *__restrict__ src, float *__restrict__ dst, int w, int h, int pitch, int newpitch)
{
  int xl = blockIdx.x * 32 + (threadIdx.x & 31);
  int yu = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (xl >= w || yu >= h) return;
  int xr = min(xl + 1, w - 1), yd = min(yu + 1, h - 1);
  float vul = __ldg(src + (size_t)yu * pitch + xl), vur = __ldg(src + (size_t)yu * pitch + xr);
  float vdl = __ldg(src + (size_t)yd * pitch + xl), vdr = __ldg(src + (size_t)yd * pitch + xr);
  float2 top = make_float2(vul, __fmul_rn(0.50f, __fadd_rn(vul, vur)));
  float2 bot = make_float2(__fmul_rn(0.50f, __fadd_rn(vul, vdl)),
                           __fmul_rn(0.25f, __fadd_rn(__fadd_rn(__fadd_rn(vul, vur), vdl), vdr)));
  float *o = dst + (size_t)(2 * yu) * newpitch + 2 * xl;
  *reinterpret_cast<float2 *>(o) = top;
  *reinterpret_cast<float2 *>(o + newpitch) = bot;
}

int launch_scaleup(const float *src, float *dst, int w, int h, int pitch, int newpitch, cudaStream_t st)
{
  dim3 grid(idivup(w, 32), idivup(h, 8));
  scaleup_kernel<<<grid, 256, 0, st>>>(src, dst, w, h, pitch, newpitch);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------
// 8-bit greyscale -> float (exact), for callers that hold camera/decoder output: uploading
// bytes moves 4x less over PCIe than the float image the reference API takes.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
u8_to_float_kernel(const uint8_t *__restrict__ src, int srcPitch, float *__restrict__ dst, int dstPitch, int w, int h)
{
  const int x = (blockIdx.x * 256 + threadIdx.x) * 4, y = blockIdx.y;
  if (x >= w || y >= h) return;
  const uint8_t *p = src + (size_t)y * srcPitch + x;
  float *o = dst + (size_t)y * dstPitch + x;
  if (x + 3 < w && ((srcPitch & 3) == 0) && ((dstPitch & 3) == 0)) {
    const uchar4 v = *reinterpret_cast<const uchar4 *>(p);
    *reinterpret_cast<float4 *>(o) = make_float4((float)v.x, (float)v.y, (float)v.z, (float)v.w);
  } else {
    for (int i = 0; i < 4 && x + i < w; i++) o[i] = (float)p[i];
  }
}

int launch_u8_to_float(const uint8_t *src, int srcPitch, float *dst, int dstPitch, int w, int h, cudaStream_t st)
{
  dim3 grid(idivup(idivup(w, 4), 256), h);
  u8_to_float_kernel<<<grid, 256, 0, st>>>(src, srcPitch, dst, dstPitch, w, h);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace cs
