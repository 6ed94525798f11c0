// common.cuh -- internal declarations shared by the cudasift_b200 translation units.
#pragma once

#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstdint>

#include "../../include/cudaSift.h"
#include "../../include/cudasift_b200.h"
#include "tma.cuh"

#define CS_NUM_SCALES 5                    // cudaSiftD.h:8
#define CS_LAPLACE_S (CS_NUM_SCALES + 3)   // 8 blurred scales -> 7 DoG planes
#define CS_MAX_LEVELS 8                    // d_PointCounter[8*2+1], cudaSiftD.cu:14

static_assert(sizeof(SiftPoint) == 576, "SiftPoint layout is ABI");
#ifdef MANAGEDMEM
static_assert(sizeof(SiftData) == 16, "SiftData layout is ABI (MANAGEDMEM flavour: numPts, maxPts, m_data)");
#else
static_assert(sizeof(SiftData) == 24, "SiftData layout is ABI");
#endif
static_assert(sizeof(CudaImage) == 48, "CudaImage layout is ABI");

namespace cs {

// ---- error handling -------------------------------------------------------------
// The C ABI reports errors through return codes + cs_last_error(); the drop-in C++ API
// keeps the reference's "message on stderr, exit(-1)" contract (cudautils.h:15-39).
void set_error(const char *fmt, ...);
extern thread_local bool g_exit_on_error;

#define CS_CUDA(call)                                                                   \
  do {                                                                                  \
    cudaError_t e_ = (call);                                                            \
    if (e_ != cudaSuccess) {                                                            \
      ::cs::set_error("%s failed at %s:%d: %s", #call, __FILE__, __LINE__,             \
                      cudaGetErrorString(e_));                                          \
      if (::cs::g_exit_on_error) {                                                      \
        fprintf(stderr, "cudasift_b200: %s\n", cs_last_error());                        \
        exit(-1);                                                                       \
      }                                                                                 \
      return CS_E_CUDA;                                                                 \
    }                                                                                   \
  } while (0)

extern unsigned long long g_launches;   // kernels launched by this library
inline void count_launch(int n = 1) { g_launches += n; }

// ---- filter taps (host) ----------------------------------------------------------
void scaledown_taps(float variance, float k[5]);                  // cudaSiftH.cu:315-324
void lowpass_taps(float sigma, float k[9]);                       // cudaSiftH.cu:408-419
void laplace_taps(int numOctaves, float initBlur, float *kernel); // cudaSiftH.cu:439-458

struct Taps9 { float k[9]; };
struct Taps5 { float k[5]; };
// [scale][tap], tap 0 = centre; every tap is stored twice (k,k): the detector consumes it as the
// uniform operand of the pair fma (tma.cuh)
struct LaplaceTaps {
  float2 k[CS_LAPLACE_S][5];
  void set(int s, int j, float v) { k[s][j].x = v; k[s][j].y = v; }
};

// ---- pyramid ----------------------------------------------------------------------
int launch_lowpass(const float *src, int srcPitch, float *dst, int dstPitch, int w, int h,
                   const Taps9 &taps, cudaStream_t st);
int launch_scaledown(const float *src, float *dst, int w, int h, int pitch, int newpitch,
                     const Taps5 &taps, cudaStream_t st, int batch = 1, long long srcStride = 0, long long dstStride = 0);
int launch_scaleup(const float *src, float *dst, int w, int h, int pitch, int newpitch,
                   cudaStream_t st);
int launch_u8_to_float(const uint8_t *src, int srcPitch, float *dst, int dstPitch, int w, int h, cudaStream_t st);

// ---- fused, batched pyramid (pyramid2.cu) ---------------------------------------------------
#define CS_MAX_BATCH 32       // images per launch (input tensor maps travel as kernel parameters)
#define CS_PA_OWN 120         // level-0 columns a warp of kernel A owns
#define CS_PA_BOX 136         // staged columns per input row (TMA box width): own + 8 left + 8 right
struct PyrAParams {
  CUtensorMap inMaps[CS_MAX_BATCH];   // input images, box 136 x 1
  float *lev0; long long lev0Stride;  // image i writes lev0 + i * lev0Stride (floats)
  float *lev1; long long lev1Stride;  // NULL: no ScaleDown (single octave)
  int w, h, p0, w1, h1, p1;
  Taps9 lp;
  Taps5 sd;
  int rowsPerCta, stripsX, rowBlocks;
};
int launch_pyr_a(const PyrAParams &p, int batch, cudaStream_t st);
const void *pyr_a_func();            // the kernel function (graph node identification)
struct PyrBParams {                   // chain of 1..3 ScaleDowns: img[0] -> img[1] -> ... -> img[steps]
  float *img[4]; long long stride[4];
  int w[4], h[4], pitch[4];
  int steps;
  Taps5 sd;
};
int launch_pyr_b(const PyrBParams &p, int batch, cudaStream_t st);

// ---- detection ---------------------------------------------------------------------
struct DetectLevel {
  const float *img;     // octave base image
  int w, h, pitch;
  float subsampling;
  float lowestScale;    // lowestScale / subsampling, cudaSiftH.cu:213
  LaplaceTaps taps;
};
struct DetectParams {
  DetectLevel lev[CS_MAX_LEVELS];
  int numLevels;
  int totalTiles;
  const uint2 *tiles;       // per tile: x = level | x0 << 8, y = y0 (built once per pipeline)
  float thresh, edgeLimit, factor;
  SiftPoint *pts;
  unsigned int *counters;   // [0] detected (primaries), [1] total incl. secondaries
  int maxPts;
};
int launch_detect(const DetectParams &p, cudaStream_t st);
#define CS_DETECT_TILE_W 62   // interior (tested) pixels per detector tile
#define CS_DETECT_TILE_H 14
int launch_dog_planes(const float *base, float *dog, int w, int h, int pitch,
                      const LaplaceTaps &taps, cudaStream_t st);

// ---- marching detector (detect2.cu): all octaves of a batch of images in one launch -----------
#define CS_CNT_STRIDE 4       // per image: [0] primaries found, [1] total incl. secondaries, [2] spare, [3] overflowed cap cells
#define CS_OVF_MAX 256        // overflowed (30x8 block, scale) cells the fix-up kernel handles per image
struct LaplaceTaps1 { float k[CS_LAPLACE_S][5]; };   // [scale][tap], tap 0 = centre
struct D2Level {
  int w, h;
  float subsampling;
  float lowestScale;          // lowestScale / subsampling, cudaSiftH.cu:213
  LaplaceTaps1 taps;
};
struct Detect2Params {
  D2Level lev[CS_MAX_LEVELS];
  const CUtensorMap *maps;    // [image * CS_MAX_LEVELS + level]: octave base images, box 256 x 1
  const uint4 *items;         // x: level | image << 8, y: x0, z: first tested row, w: rows per stream
  int numItems;
  float thresh, edgeLimit, factor;
  SiftPoint *pts;             // image i writes pts + i * ptsStride
  long long ptsStride;        // in records
  unsigned int *counters;     // image i: counters + i * CS_CNT_STRIDE
  unsigned int *sched;        // dynamic item scheduler (zeroed before the launch)
  int maxPts;
  // reference cap of 32 extrema per 30x8 block and scale (cudaSiftD.cu:1371,1379); cells == NULL: no cap
  unsigned int *cells;        // packed 8-bit counters, image i: cells + i * cellWords
  int cellWords;
  int capLimit;               // 32 (MEMWID, cudaSiftD.cu:1293); tests lower it to make the cap reachable
  int cellBase[CS_MAX_LEVELS], cellsX[CS_MAX_LEVELS];
  const float *lev0Img[CS_MAX_LEVELS];   // level images of image slot 0 (fix-up kernel): slot i at + i * imgStride
  long long imgStride;
  int levPitch[CS_MAX_LEVELS];
};
int launch_detect2(const Detect2Params &p, int sms, cudaStream_t st);
int detect2_init_device();   // fills the device-side pow table (once per device; not inside a stream capture)
int launch_cap32_fixup(const Detect2Params &p, int batch, cudaStream_t st);
#define CS_D2_STRIP 244       // tested columns per detector strip (multiple of 4: TMA box alignment)

// ---- orientation + descriptor ---------------------------------------------------------
struct DescribeParams {
  cudaTextureObject_t tex[CS_MAX_LEVELS];   // indexed by log2(subsampling); used when texArr == NULL
  const cudaTextureObject_t *texArr;        // batch: [image * CS_MAX_LEVELS + level] (device memory)
  int numLevels;
  SiftPoint *pts;                           // image i: pts + i * ptsStride
  long long ptsStride;
  unsigned int *counters;                   // image i: counters + i * cntStride
  int cntStride;
  int maxPts;
  float finestSubsampling;  // secondaries of this level are dropped (reference quirk Q1)
};
int launch_describe(const DescribeParams &p, int gridBlocks, cudaStream_t st, int batch = 1);
int launch_rescale(SiftPoint *pts, const unsigned int *counters, int maxPts, float f,
                   cudaStream_t st);
int launch_tex_probe(cudaTextureObject_t tex, const float *xs, const float *ys, int n,
                     float *out, cudaStream_t st);

int make_texture(cudaTextureObject_t *tex, const float *img, int w, int h, int pitch);

// ---- ranking (rank.cu): per image the maxOut candidates with the largest |sharpness|, in key order ---------------
#define CS_RANK_MAX_IN (1 << 18)    // largest candidate count per image
#define CS_RANK_SCRATCH_PER_IN 9    // scratch words per candidate
struct RankParams {
  const SiftPoint *in; long long inStride;   // image i: candidates in + i * inStride, count read from its counters
  SiftPoint *out; long long outStride;       // image i: min(maxOut, found) records in rank order
  unsigned int *counters;                    // image i: counters + i * CS_CNT_STRIDE; [2] receives the output count
  unsigned int *scratch;                     // image i: scratch + i * rank_scratch_words(maxIn)
  int maxIn, maxOut;
};
// per image: [maxIn] primary keys | [7][maxIn] survivors' keys and candidate index | [maxIn] survivors' ranks
// | survivor count (4 words)
__host__ __device__ inline size_t rank_scratch_words(int maxIn)
{
  return (size_t)maxIn * CS_RANK_SCRATCH_PER_IN + 4;
}
int launch_rank(const RankParams &p, int batch, int sms, cudaStream_t st);

// ---- matcher ------------------------------------------------------------------------
struct MatchWorkspace;   // opaque, owned by the per-device context
int match_exact(SiftPoint *s1, int n1, const SiftPoint *s2, int n2, cudaStream_t st);
int match_tensor(SiftPoint *s1, int n1, const SiftPoint *s2, int n2, cudaStream_t st,
                 unsigned long long stats[4]);
bool match_tensor_supported();
void match_tensor_stats(unsigned long long stats[4]);   // after a synchronize

inline int idivup(int a, int b) { return (a + b - 1) / b; }
inline int ialignup(int a, int b) { return (a % b != 0) ? (a - a % b + b) : a; }

}  // namespace cs
