// api.cu -- host side of libcudasift_b200.so: the drop-in C++ API of the reference
// (cudaSift.h / cudaImage.h: InitCuda, ExtractSift, MatchSiftData, CudaImage ...) and the
// additive C ABI declared in include/cudasift_b200.h.
//
// Reference host code this replaces: cudaSiftH.cu:19-302 (driver, temp memory, SiftData),
// cudaSiftH.cu:308-514 (per-stage launchers), cudaImage.cu:10-115, matching.cu:1090-1206.
// Differences in structure (not in results): one stream-ordered pipeline of 8 launches per
// image instead of 25 launches with 4 blocking copies and 5 texture create/destroy pairs;
// per-device state instead of function-local statics (quirk Q12); quiet unless
// CUDASIFT_VERBOSE is set (quirk Q13).
#include "common.cuh"
#include "pipeline2.h"

#include <cmath>
#include <cstdarg>
#include <cstring>
#include <chrono>
#include <map>
#include <mutex>
#include <vector>

namespace cs {

// ------------------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";
thread_local bool g_exit_on_error = false;
unsigned long long g_launches = 0;

void set_error(const char *fmt, ...)
{
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// CUDASIFT_LEGACY=1 (or cs_set_tuning("legacy", 1)): the round-1 per-image kernels instead of the batched
// TMA pipeline.  The legacy path is also what an image that TMA cannot address (odd pitch, unaligned base) takes.
int g_legacy = -1;
static bool legacy_mode()
{
  if (g_legacy < 0) { const char *e = getenv("CUDASIFT_LEGACY"); g_legacy = (e && *e && *e != '0') ? 1 : 0; }
  return g_legacy == 1;
}

static bool verbose()
{
  static int v = -1;
  if (v < 0) { const char *e = getenv("CUDASIFT_VERBOSE"); v = (e && *e && *e != '0') ? 1 : 0; }
  return v == 1;
}

// ------------------------------------------------------------------------------ taps
void scaledown_taps(float variance, float k[5])
{ // cudaSiftH.cu:315-324
  float sum = 0.0f;
  for (int j = 0; j < 5; j++) {
    k[j] = (float)expf(-(double)(j - 2) * (j - 2) / 2.0 / variance);
    sum += k[j];
  }
  for (int j = 0; j < 5; j++) k[j] /= sum;
}

void lowpass_taps(float sigma, float k[9])
{ // cudaSiftH.cu:408-419
  float sum = 0.0f;
  float ivar2 = 1.0f / (2.0f * sigma * sigma);
  for (int j = -4; j <= 4; j++) {
    k[j + 4] = (float)expf(-(double)j * j * ivar2);
    sum += k[j + 4];
  }
  for (int j = -4; j <= 4; j++) k[j + 4] /= sum;
}

void laplace_taps(int numOctaves, float initBlur, float *kernel)
{ // cudaSiftH.cu:439-458
  if (numOctaves > 1) {
    float totInitBlur = (float)sqrtf(initBlur * initBlur + 0.5f * 0.5f) / 2.0f;
    laplace_taps(numOctaves - 1, totInitBlur, kernel);
  }
  float scale = powf(2.0f, -1.0f / CS_NUM_SCALES);
  float diffScale = powf(2.0f, 1.0f / CS_NUM_SCALES);
  for (int i = 0; i < CS_NUM_SCALES + 3; i++) {
    float sum = 0.0f;
    float var = scale * scale - initBlur * initBlur;
    float *k = kernel + numOctaves * 12 * 16 + 16 * i;
    for (int j = 0; j <= 4; j++) {
      k[j] = (float)expf(-(double)j * j / 2.0 / var);
      sum += (j == 0 ? 1 : 2) * k[j];
    }
    for (int j = 0; j <= 4; j++) k[j] /= sum;
    scale *= diffScale;
  }
}

// --------------------------------------------------------------------- temp memory sizing
static size_t temp_floats(int width, int height, int numOctaves, bool scaleUp)
{ // cudaSiftH.cu:39-57 (same rule, so arenas are interchangeable with the reference's)
  const int nd = CS_NUM_SCALES + 3;
  int w = width * (scaleUp ? 2 : 1), h = height * (scaleUp ? 2 : 1);
  int p = ialignup(w, 128);
  size_t size = (size_t)h * p, sizeTmp = (size_t)nd * h * p;
  for (int i = 0; i < numOctaves; i++) {
    w /= 2; h /= 2;
    int pp = ialignup(w, 128);
    size += (size_t)h * pp;
    sizeTmp += (size_t)nd * h * pp;
  }
  return size + sizeTmp;
}

// ------------------------------------------------------------------------------ pipeline
// One Pipeline = everything ExtractSift needs for one (width, height, octaves, scaleUp,
// arena) combination: level pointers inside the arena, texture objects, counters.
struct Pipeline {
  int w0 = 0, h0 = 0, numOctaves = 0;
  bool scaleUp = false;
  float *arena = nullptr;
  bool ownArena = false;
  int numLevels = 0;
  float *lev[CS_MAX_LEVELS] = {};
  int lw[CS_MAX_LEVELS] = {}, lh[CS_MAX_LEVELS] = {}, lp[CS_MAX_LEVELS] = {};
  float *upImg = nullptr;
  cudaTextureObject_t tex[CS_MAX_LEVELS] = {};
  unsigned int *d_counters = nullptr;   // [0] primaries found, [1] total incl. secondaries
  uint2 *d_tiles = nullptr;             // detector tile list (level, x0, y0), all levels
  int numTiles = 0;
  float lapTaps[8 * 12 * 16];
  Taps5 sdTaps;
  int describeBlocks = 0;

  int init(int w, int h, int octaves, bool up, float *arenaPtr);
  void destroy();
  // ev (optional): 5 events recorded at stage boundaries (start, after LowPass, after the
  // ScaleDown chain, after detect, after describe) for per-kernel timing.
  int enqueue(const float *d_img, int pitch, double initBlur, float thresh, float lowestScale,
              SiftPoint *d_pts, int maxPts, cudaStream_t st, cudaEvent_t *ev = nullptr);
};

int Pipeline::init(int w, int h, int octaves, bool up, float *arenaPtr)
{
  if (w < 1 || h < 1 || octaves < 1 || octaves > 7) {   // quirk Q17: taps table holds octave <= 7
    set_error("ExtractSift: invalid size %dx%d or numOctaves %d (1..7)", w, h, octaves);
    return CS_E_ARG;
  }
  w0 = w; h0 = h; numOctaves = octaves; scaleUp = up;
  if (arenaPtr) { arena = arenaPtr; ownArena = false; }
  else {
    size_t fl = temp_floats(w, h, octaves, up);
    CS_CUDA(cudaMalloc((void **)&arena, fl * sizeof(float)));
    ownArena = true;
  }
  int W = w * (up ? 2 : 1), H = h * (up ? 2 : 1);
  float *cur = arena;
  numLevels = octaves;
  lw[0] = W; lh[0] = H; lp[0] = ialignup(W, 128);
  for (int i = 0; i < octaves; i++) {
    if (i > 0) { lw[i] = lw[i - 1] / 2; lh[i] = lh[i - 1] / 2; lp[i] = ialignup(lw[i], 128); }
    lev[i] = cur;
    cur += (size_t)lh[i] * lp[i];
    if (lw[i] < 1 || lh[i] < 1) { numLevels = i; break; }
  }
  if (up) { upImg = cur; cur += (size_t)lh[0] * lp[0]; }
  for (int i = 0; i < numLevels; i++) {
    int r = make_texture(&tex[i], lev[i], lw[i], lh[i], lp[i]);
    if (r < 0) return r;
  }
  CS_CUDA(cudaMalloc((void **)&d_counters, 4 * sizeof(unsigned int)));
  {
    // coarsest level first: its tiles carry the most extrema candidates, so the persistent CTAs
    // finish on the light tiles of the finest level
    std::vector<uint2> tl;
    int nl = 0, idx[CS_MAX_LEVELS];
    for (int i = 0; i < numLevels; i++) idx[i] = (lw[i] < 3 || lh[i] < 3) ? -1 : nl++;   // no interior pixel -> no extrema
    for (int i = numLevels - 1; i >= 0; i--) {
      if (idx[i] < 0) continue;
      const int tx = idivup(lw[i] - 2, CS_DETECT_TILE_W), ty = idivup(lh[i] - 2, CS_DETECT_TILE_H);
      for (int y = 0; y < ty; y++)
        for (int x = 0; x < tx; x++)
          tl.push_back(make_uint2((unsigned)idx[i] | ((unsigned)(x * CS_DETECT_TILE_W) << 8), (unsigned)(y * CS_DETECT_TILE_H)));
    }
    numTiles = (int)tl.size();
    if (numTiles > 0) {
      CS_CUDA(cudaMalloc((void **)&d_tiles, tl.size() * sizeof(uint2)));
      CS_CUDA(cudaMemcpy(d_tiles, tl.data(), tl.size() * sizeof(uint2), cudaMemcpyHostToDevice));
    }
  }
  memset(lapTaps, 0, sizeof(lapTaps));
  laplace_taps(octaves, 0.0f, lapTaps);           // cudaSiftH.cu:110
  scaledown_taps(0.5f, sdTaps.k);                 // cudaSiftH.cu:157
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  describeBlocks = sms * 8;
  return 0;
}

void Pipeline::destroy()
{
  for (int i = 0; i < CS_MAX_LEVELS; i++)
    if (tex[i]) { cudaDestroyTextureObject(tex[i]); tex[i] = 0; }
  if (d_counters) { cudaFree(d_counters); d_counters = nullptr; }
  if (d_tiles) { cudaFree(d_tiles); d_tiles = nullptr; }
  if (ownArena && arena) cudaFree(arena);
  arena = nullptr;
}

int Pipeline::enqueue(const float *d_img, int pitch, double initBlur, float thresh, float lowestScale,
                      SiftPoint *d_pts, int maxPts, cudaStream_t st, cudaEvent_t *ev)
{
  int r;
  CS_CUDA(cudaMemsetAsync(d_counters, 0, 4 * sizeof(unsigned int), st));   // cudaSiftH.cu:77
  if (ev) cudaEventRecord(ev[0], st);
  Taps9 lp9;
  float sigma = (float)(initBlur > (double)0.001f ? initBlur : (double)0.001f);   // cudaSiftH.cu:112
  lowpass_taps(sigma, lp9.k);
  if (!scaleUp) {
    if ((r = launch_lowpass(d_img, pitch, lev[0], lp[0], lw[0], lh[0], lp9, st)) < 0) return r;
  } else {                                                                 // cudaSiftH.cu:119-123
    if ((r = launch_scaleup(d_img, upImg, w0, h0, pitch, lp[0], st)) < 0) return r;
    if ((r = launch_lowpass(upImg, lp[0], lev[0], lp[0], lw[0], lh[0], lp9, st)) < 0) return r;
    lowestScale *= 2.0f;                                                   // cudaSiftH.cu:127
  }
  if (ev) cudaEventRecord(ev[1], st);
  for (int i = 1; i < numLevels; i++)                                      // cudaSiftH.cu:153-157
    if ((r = launch_scaledown(lev[i - 1], lev[i], lw[i - 1], lh[i - 1], lp[i - 1], lp[i], sdTaps, st)) < 0) return r;
  if (ev) cudaEventRecord(ev[2], st);

  DetectParams dp;
  memset(&dp, 0, sizeof(dp));
  int tiles = 0, nl = 0;
  for (int i = 0; i < numLevels; i++) {
    if (lw[i] < 3 || lh[i] < 3) continue;          // no interior pixel -> no extrema possible
    DetectLevel &L = dp.lev[nl++];
    L.img = lev[i]; L.w = lw[i]; L.h = lh[i]; L.pitch = lp[i];
    tiles += idivup(lw[i] - 2, CS_DETECT_TILE_W) * idivup(lh[i] - 2, CS_DETECT_TILE_H);   // see Pipeline::init (d_tiles)
    L.subsampling = (float)(1 << i);
    L.lowestScale = lowestScale / L.subsampling;                           // cudaSiftH.cu:213
    const float *k = lapTaps + (numOctaves - i) * 12 * 16;                 // octave index, :161,:1766
    for (int s = 0; s < CS_LAPLACE_S; s++)
      for (int j = 0; j < 5; j++) L.taps.set(s, j, k[16 * s + j]);
  }
  dp.numLevels = nl; dp.totalTiles = tiles; dp.tiles = d_tiles;
  if (tiles != numTiles) { set_error("detector tile list out of sync"); return CS_E_ARG; }
  dp.thresh = thresh; dp.edgeLimit = 10.0f; dp.factor = 1.0f / CS_NUM_SCALES;   // cudaSiftH.cu:213
  dp.pts = d_pts; dp.counters = d_counters; dp.maxPts = maxPts;
  if ((r = launch_detect(dp, st)) < 0) return r;
  if (ev) cudaEventRecord(ev[3], st);

  DescribeParams ds;
  memset(&ds, 0, sizeof(ds));
  for (int i = 0; i < numLevels; i++) ds.tex[i] = tex[i];
  ds.numLevels = numLevels; ds.pts = d_pts; ds.counters = d_counters; ds.maxPts = maxPts;
  ds.finestSubsampling = 1.0f;
  if ((r = launch_describe(ds, describeBlocks, st)) < 0) return r;
  if (scaleUp)                                                             // cudaSiftH.cu:130
    if ((r = launch_rescale(d_pts, d_counters, maxPts, 0.5f, st)) < 0) return r;
  if (ev) cudaEventRecord(ev[4], st);
  return 0;
}

static inline int count_from_counters(const unsigned int *c, int maxPts)
{
  unsigned int a = c[0] < (unsigned)maxPts ? c[0] : (unsigned)maxPts;
  unsigned int b = c[1] < (unsigned)maxPts ? c[1] : (unsigned)maxPts;
  return (int)(a > b ? a : b);
}

// ------------------------------------------------------------------------------ device ctx
struct PipeKey {
  int w, h, oct, up; float *arena;
  bool operator<(const PipeKey &o) const
  {
    if (w != o.w) return w < o.w;
    if (h != o.h) return h < o.h;
    if (oct != o.oct) return oct < o.oct;
    if (up != o.up) return up < o.up;
    return arena < o.arena;
  }
};

struct DeviceCtx {
  int dev = -1;
  cudaStream_t stream = nullptr;           // blocking stream: ordered after legacy default-stream work
  std::map<PipeKey, Pipeline *> pipes;     // legacy per-image pipelines
  std::map<PipeKey, Pipeline2 *> pipes2;   // batched pipeline, batch of one (the drop-in ExtractSift)
  unsigned int *h_counters = nullptr;      // pinned
  unsigned long long matchStats[4] = {0, 0, 0, 0};
  // scratch for *_host entry points
  void *scratch[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};   // 4: cs_rank_records
  size_t scratchBytes[5] = {0, 0, 0, 0, 0};

  int ensure(int d)
  {
    if (dev == d && stream) return 0;
    dev = d;
    CS_CUDA(cudaStreamCreate(&stream));
    CS_CUDA(cudaMallocHost((void **)&h_counters, 4 * sizeof(unsigned int)));
    return 0;
  }
  int get_scratch(int slot, size_t bytes, void **out)
  {
    if (scratchBytes[slot] < bytes) {
      if (scratch[slot]) cudaFree(scratch[slot]);
      scratch[slot] = nullptr; scratchBytes[slot] = 0;
      CS_CUDA(cudaMalloc(&scratch[slot], bytes));
      scratchBytes[slot] = bytes;
    }
    *out = scratch[slot];
    return 0;
  }
  Pipeline *get_pipe(int w, int h, int oct, bool up, float *arena, int *err)
  {
    PipeKey k{w, h, oct, up ? 1 : 0, arena};
    auto it = pipes.find(k);
    if (it != pipes.end()) return it->second;
    if (!arena && pipes.size() > 8) drop_pipes(nullptr, true);   // bound the internal-arena cache
    Pipeline *p = new Pipeline();
    int r = p->init(w, h, oct, up, arena);
    if (r < 0) { p->destroy(); delete p; *err = r; return nullptr; }
    pipes[k] = p;
    return p;
  }
  Pipeline2 *get_pipe2(int w, int h, int oct, bool up, float *arena, int *err)
  {
    PipeKey k{w, h, oct, up ? 1 : 0, arena};
    auto it = pipes2.find(k);
    if (it != pipes2.end()) return it->second;
    if (!arena && pipes2.size() > 8) drop_pipes(nullptr, true);
    Pipeline2 *p = new Pipeline2();
    int r = p->init(w, h, oct, up, 1, arena);
    if (r < 0) { p->destroy(); delete p; *err = r; return nullptr; }
    pipes2[k] = p;
    return p;
  }
  void drop_pipes(float *arena, bool internalOnly)
  {
    for (auto it = pipes.begin(); it != pipes.end();) {
      bool hit = internalOnly ? it->second->ownArena : (it->first.arena == arena);
      if (hit) { it->second->destroy(); delete it->second; it = pipes.erase(it); }
      else ++it;
    }
    for (auto it = pipes2.begin(); it != pipes2.end();) {
      bool hit = internalOnly ? it->second->ownArena : (it->first.arena == arena);
      if (hit) { it->second->destroy(); delete it->second; it = pipes2.erase(it); }
      else ++it;
    }
  }
};

static std::mutex g_mutex;
static std::map<int, DeviceCtx *> g_ctx;

static DeviceCtx *current_ctx(int *err)
{
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    set_error("no usable CUDA device (%s): cudasift_b200 has no CPU fallback", cudaGetErrorString(e));
    *err = CS_E_NODEV;
    if (g_exit_on_error) { fprintf(stderr, "cudasift_b200: %s\n", g_err); exit(-1); }
    return nullptr;
  }
  std::lock_guard<std::mutex> lk(g_mutex);
  DeviceCtx *&c = g_ctx[dev];
  if (!c) c = new DeviceCtx();
  int r = c->ensure(dev);
  if (r < 0) { *err = r; return nullptr; }
  return c;
}

// ------------------------------------------------------------------------------ core ops
static int extract_sync(const float *d_img, int w, int h, int pitch, int numOctaves, double initBlur,
                        float thresh, float lowestScale, bool scaleUp, float *d_tmp, SiftPoint *d_pts,
                        SiftPoint *h_pts, int maxPts, double *msKernel)
{
  int err = 0;
  if (!d_img || !d_pts || maxPts < 1) { set_error("ExtractSift: missing image or SiftData"); return CS_E_ARG; }
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const bool useLegacy = legacy_mode() || !tensor_map_compatible(d_img, pitch) ||
                         (d_tmp && (reinterpret_cast<uintptr_t>(d_tmp) & 15) != 0);
  Pipeline *p = nullptr;
  Pipeline2 *p2 = nullptr;
  if (useLegacy) p = c->get_pipe(w, h, numOctaves, scaleUp, d_tmp, &err);
  else p2 = c->get_pipe2(w, h, numOctaves, scaleUp, d_tmp, &err);
  if (!p && !p2) return err;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (msKernel) { cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventRecord(e0, c->stream); }
  int r = p ? p->enqueue(d_img, pitch, initBlur, thresh, lowestScale, d_pts, maxPts, c->stream)
            : p2->enqueue(1, &d_img, pitch, initBlur, thresh, lowestScale, d_pts, 0, maxPts, c->stream);
  if (r < 0) { if (msKernel) { cudaEventDestroy(e0); cudaEventDestroy(e1); } return r; }
  if (msKernel) cudaEventRecord(e1, c->stream);
  const unsigned int *d_cnt = p ? p->d_counters : p2->counters(0);
  CS_CUDA(cudaMemcpyAsync(c->h_counters, d_cnt, 2 * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
  CS_CUDA(cudaStreamSynchronize(c->stream));
  int numPts = count_from_counters(c->h_counters, maxPts);                 // cudaSiftH.cu:115-116
  if (msKernel) {
    float ms = 0; cudaEventElapsedTime(&ms, e0, e1); *msKernel = ms;
    cudaEventDestroy(e0); cudaEventDestroy(e1);
  }
  if (h_pts && numPts > 0) {                                               // cudaSiftH.cu:139-140
    CS_CUDA(cudaMemcpyAsync(h_pts, d_pts, sizeof(SiftPoint) * (size_t)numPts, cudaMemcpyDeviceToHost, c->stream));
    CS_CUDA(cudaStreamSynchronize(c->stream));
  }
  return numPts;
}

static int match_sync(SiftPoint *d_s1, int n1, SiftPoint *d_s2, int n2, SiftPoint *h_s1, int mode, double *ms)
{
  int err = 0;
  if (ms) *ms = 0.0;
  if (!n1 || !n2) return 0;                                                // matching.cu:1095-1096
  if (!d_s1 || !d_s2) return 0;                                            // matching.cu:1101-1102
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0, c->stream);
  int r;
  bool useTensor = (mode == 2) || (mode == 0 && match_tensor_supported() && n1 >= 256 && n2 >= 256);
  if (useTensor) {
    r = match_tensor(d_s1, n1, d_s2, n2, c->stream, c->matchStats);
    c->matchStats[3] = 2;
  } else {
    r = match_exact(d_s1, n1, d_s2, n2, c->stream);
    c->matchStats[0] = c->matchStats[1] = c->matchStats[2] = 0; c->matchStats[3] = 1;
  }
  if (r >= 0 && h_s1) {                                                    // matching.cu:1195-1199
    cudaError_t ce = cudaMemcpy2DAsync(&h_s1[0].score, sizeof(SiftPoint), &d_s1[0].score, sizeof(SiftPoint),
                                       5 * sizeof(float), n1, cudaMemcpyDeviceToHost, c->stream);
    if (ce != cudaSuccess) { set_error("MatchSiftData: result copy failed: %s", cudaGetErrorString(ce)); r = CS_E_CUDA; }
  }
  if (r >= 0) {
    cudaEventRecord(e1, c->stream);
    cudaError_t ce = cudaStreamSynchronize(c->stream);
    if (ce != cudaSuccess) { set_error("MatchSiftData: %s", cudaGetErrorString(ce)); r = CS_E_CUDA; }
  }
  if (r < 0) { cudaEventDestroy(e0); cudaEventDestroy(e1); return r; }     // no event leak on the error paths
  float t = 0; cudaEventElapsedTime(&t, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  if (useTensor) match_tensor_stats(c->matchStats);
  if (ms) *ms = t;
  return 0;
}

}  // namespace cs

using namespace cs;

// =====================================================================================
// Drop-in C++ API (same mangled symbols as the reference objects)
// =====================================================================================
struct ExitGuard {
  bool prev;
  ExitGuard() : prev(g_exit_on_error) { g_exit_on_error = true; }
  ~ExitGuard() { g_exit_on_error = prev; }
};

static void die_if(int r)
{
  if (r < 0) { fprintf(stderr, "cudasift_b200: %s\n", cs_last_error()); exit(-1); }
}

int iDivUp(int a, int b) { return (a % b != 0) ? (a / b + 1) : (a / b); }
int iDivDown(int a, int b) { return a / b; }
int iAlignUp(int a, int b) { return (a % b != 0) ? (a - a % b + b) : a; }
int iAlignDown(int a, int b) { return a - a % b; }

static std::chrono::steady_clock::time_point g_timers[16];
void StartTimer(unsigned int *hTimer)
{
  static unsigned int next = 0;
  unsigned int id = (next++) & 15;
  g_timers[id] = std::chrono::steady_clock::now();
  if (hTimer) *hTimer = id;
}
double StopTimer(unsigned int hTimer)
{
  auto d = std::chrono::steady_clock::now() - g_timers[hTimer & 15];
  return std::chrono::duration<double, std::milli>(d).count();
}

CudaImage::CudaImage()
    : width(0), height(0), pitch(0), h_data(NULL), d_data(NULL), t_data(NULL), d_internalAlloc(false),
      h_internalAlloc(false) {}

CudaImage::~CudaImage()
{ // cudaImage.cu:42-53
  if (d_internalAlloc && d_data != NULL) cudaFree(d_data);
  d_data = NULL;
  if (h_internalAlloc && h_data != NULL) free(h_data);
  h_data = NULL;
  if (t_data != NULL) cudaFreeArray((cudaArray *)t_data);
  t_data = NULL;
}

void CudaImage::Allocate(int w, int h, int p, bool host, float *devmem, float *hostmem)
{ // cudaImage.cu:15-34 (without the int* -> size_t* cast of quirk Q20)
  ExitGuard g;
  width = w; height = h; pitch = p;
  d_data = devmem; h_data = hostmem; t_data = NULL;
  if (devmem == NULL) {
    size_t pitchBytes = 0;
    cudaError_t e = cudaMallocPitch((void **)&d_data, &pitchBytes, sizeof(float) * (size_t)width, (size_t)height);
    if (e != cudaSuccess) { fprintf(stderr, "cudasift_b200: cudaMallocPitch failed: %s\n", cudaGetErrorString(e)); exit(-1); }
    pitch = (int)(pitchBytes / sizeof(float));
    d_internalAlloc = true;
  }
  if (host && hostmem == NULL) {
    h_data = (float *)malloc(sizeof(float) * (size_t)pitch * height);
    h_internalAlloc = true;
  }
}

static double ms_since(std::chrono::steady_clock::time_point t0)
{
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

double CudaImage::Download()
{ // cudaImage.cu:55-66
  auto t0 = std::chrono::steady_clock::now();
  if (d_data != NULL && h_data != NULL) {
    cudaError_t e = cudaMemcpy2D(d_data, sizeof(float) * pitch, h_data, sizeof(float) * width, sizeof(float) * width,
                                 height, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { fprintf(stderr, "cudasift_b200: Download failed: %s\n", cudaGetErrorString(e)); exit(-1); }
  }
  return ms_since(t0);
}

double CudaImage::Readback()
{ // cudaImage.cu:68-78
  auto t0 = std::chrono::steady_clock::now();
  cudaError_t e = cudaMemcpy2D(h_data, sizeof(float) * width, d_data, sizeof(float) * pitch, sizeof(float) * width,
                               height, cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) { fprintf(stderr, "cudasift_b200: Readback failed: %s\n", cudaGetErrorString(e)); exit(-1); }
  return ms_since(t0);
}

double CudaImage::InitTexture()
{ // cudaImage.cu:80-92 (legacy cudaArray helper, unused by the extraction path)
  auto t0 = std::chrono::steady_clock::now();
  cudaChannelFormatDesc desc = cudaCreateChannelDesc<float>();
  cudaError_t e = cudaMallocArray((cudaArray **)&t_data, &desc, pitch, height);
  if (e != cudaSuccess || t_data == NULL) printf("Failed to allocated texture data\n");
  return ms_since(t0);
}

double CudaImage::CopyToTexture(CudaImage &dst, bool host)
{ // cudaImage.cu:94-115
  if (dst.t_data == NULL) { printf("Error CopyToTexture: No texture data\n"); return 0.0; }
  if ((!host || h_data == NULL) && (host || d_data == NULL)) { printf("Error CopyToTexture: No source data\n"); return 0.0; }
  auto t0 = std::chrono::steady_clock::now();
  const float *src = host ? h_data : d_data;
  cudaMemcpy2DToArray((cudaArray *)dst.t_data, 0, 0, src, sizeof(float) * pitch, sizeof(float) * pitch, dst.height,
                      host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice);
  cudaDeviceSynchronize();
  return ms_since(t0);
}

void InitCuda(int devNum)
{ // cudaSiftH.cu:19-37
  ExitGuard g;
  die_if(cs_init(devNum) < 0 ? -1 : 0);
}

float *AllocSiftTempMemory(int width, int height, int numOctaves, bool scaleUp)
{
  ExitGuard g;
  float *p = cs_alloc_temp(width, height, numOctaves, scaleUp ? 1 : 0);
  if (!p) die_if(-1);
  return p;
}

void FreeSiftTempMemory(float *memoryTmp) { cs_free_temp(memoryTmp); }

void ExtractSift(SiftData &siftData, CudaImage &img, int numOctaves, double initBlur, float thresh,
                 float lowestScale, bool scaleUp, float *tempMemory)
{ // cudaSiftH.cu:72-144
  ExitGuard g;
  auto t0 = std::chrono::steady_clock::now();
  double msK = 0.0;
#ifdef MANAGEDMEM
  SiftPoint *d = siftData.m_data, *hh = NULL;
#else
  SiftPoint *d = siftData.d_data, *hh = siftData.h_data;
#endif
  int n = extract_sync(img.d_data, img.width, img.height, img.pitch, numOctaves, initBlur, thresh, lowestScale,
                       scaleUp, tempMemory, d, hh, siftData.maxPts, verbose() ? &msK : NULL);
  die_if(n);
  siftData.numPts = n;
  if (verbose()) {
    printf("SIFT extraction time =        %.2f ms %d\n", msK, siftData.numPts);
    printf("Incl prefiltering & memcpy =  %.2f ms %d\n\n", ms_since(t0), siftData.numPts);
  }
}

// ---- stage-level host entry points of the reference (cudaSiftH.h:11-22) ----------------
// Same signatures and mangled names; mainSift.cpp:20 declares ScaleUp itself.
double ScaleUp(CudaImage &res, CudaImage &src)
{ // cudaSiftH.cu:340-351
  if (res.d_data == NULL || src.d_data == NULL) { printf("ScaleUp: missing data\n"); return 0.0; }
  ExitGuard g;
  die_if(cs_scaleup(src.d_data, res.d_data, src.width, src.height, src.pitch, res.pitch));
  return 0.0;
}

double ScaleDown(CudaImage &res, CudaImage &src, float variance)
{ // cudaSiftH.cu:308-338
  if (res.d_data == NULL || src.d_data == NULL) { printf("ScaleDown: missing data\n"); return 0.0; }
  ExitGuard g;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  die_if(c ? 0 : err);
  Taps5 t; scaledown_taps(variance, t.k);
  die_if(launch_scaledown(src.d_data, res.d_data, src.width, src.height, src.pitch, res.pitch, t, c->stream));
  cudaStreamSynchronize(c->stream);
  return 0.0;
}

double LowPass(CudaImage &res, CudaImage &src, float scale)
{ // cudaSiftH.cu:406-435
  ExitGuard g;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  die_if(c ? 0 : err);
  Taps9 t; lowpass_taps(scale, t.k);
  die_if(launch_lowpass(src.d_data, src.pitch, res.d_data, res.pitch, res.width, res.height, t, c->stream));
  cudaStreamSynchronize(c->stream);
  return 0.0;
}

void PrepareLaplaceKernels(int numOctaves, float initBlur, float *kernel)
{ // cudaSiftH.cu:439-458
  laplace_taps(numOctaves, initBlur, kernel);
}

void InitSiftData(SiftData &data, int num, bool host, bool dev)
{ // cudaSiftH.cu:234-249
  ExitGuard g;
  data.numPts = 0;
  data.maxPts = num;
  size_t sz = sizeof(SiftPoint) * (size_t)num;
#ifdef MANAGEDMEM
  if (cudaMallocManaged((void **)&data.m_data, sz) != cudaSuccess) die_if(-1);
#else
  data.h_data = NULL;
  if (host) data.h_data = (SiftPoint *)malloc(sz);
  data.d_data = NULL;
  if (dev) {
    cudaError_t e = cudaMalloc((void **)&data.d_data, sz);
    if (e != cudaSuccess) { set_error("InitSiftData: cudaMalloc(%zu) failed: %s", sz, cudaGetErrorString(e)); die_if(-1); }
  }
#endif
}

void FreeSiftData(SiftData &data)
{ // cudaSiftH.cu:251-264
#ifdef MANAGEDMEM
  cudaFree(data.m_data);
#else
  if (data.d_data != NULL) cudaFree(data.d_data);
  data.d_data = NULL;
  if (data.h_data != NULL) free(data.h_data);
  data.h_data = NULL;
#endif
  data.numPts = 0;
  data.maxPts = 0;
}

void PrintSiftData(SiftData &data)
{ // cudaSiftH.cu:266-302
#ifdef MANAGEDMEM
  SiftPoint *h = data.m_data;
#else
  SiftPoint *h = data.h_data;
  if (h == NULL) {
    h = (SiftPoint *)malloc(sizeof(SiftPoint) * (size_t)data.maxPts);
    cudaMemcpy(h, data.d_data, sizeof(SiftPoint) * (size_t)data.numPts, cudaMemcpyDeviceToHost);
    data.h_data = h;
  }
#endif
  for (int i = 0; i < data.numPts; i++) {
    printf("xpos         = %.2f\n", h[i].xpos);
    printf("ypos         = %.2f\n", h[i].ypos);
    printf("scale        = %.2f\n", h[i].scale);
    printf("sharpness    = %.2f\n", h[i].sharpness);
    printf("edgeness     = %.2f\n", h[i].edgeness);
    printf("orientation  = %.2f\n", h[i].orientation);
    printf("score        = %.2f\n", h[i].score);
    const float *v = h[i].data;
    for (int j = 0; j < 8; j++) {
      printf(j == 0 ? "data = " : "       ");
      for (int k = 0; k < 16; k++) {
        if (v[j + 8 * k] < 0.05) printf(" .   ");
        else printf("%.2f ", v[j + 8 * k]);
      }
      printf("\n");
    }
  }
  printf("Number of available points: %d\n", data.numPts);
  printf("Number of allocated points: %d\n", data.maxPts);
}

double MatchSiftData(SiftData &data1, SiftData &data2)
{ // matching.cu:1090-1206
  ExitGuard g;
  double ms = 0.0;
#ifdef MANAGEDMEM
  int r = match_sync(data1.m_data, data1.numPts, data2.m_data, data2.numPts, NULL, 0, &ms);
#else
  int r = match_sync(data1.d_data, data1.numPts, data2.d_data, data2.numPts, data1.h_data, 0, &ms);
#endif
  die_if(r);
  if (verbose()) printf("MatchSiftData time =          %.2f ms\n", ms);
  return ms;
}

// =====================================================================================
// C ABI
// =====================================================================================
extern "C" {

const char *cs_last_error(void) { return cs::g_err; }
const char *cs_version(void) { return "cudasift_b200 0.1 (sm_90a)"; }
unsigned long long cs_launch_count(void) { return cs::g_launches; }

int cs_set_tuning(const char *key, int value)
{
  if (key && strcmp(key, "legacy") == 0) { cs::g_legacy = value ? 1 : 0; return 0; }
  if (key && strcmp(key, "d2_hs") == 0) { cs::g_d2_hs = value; return 0; }
  if (key && strcmp(key, "pa_rows") == 0) { cs::g_pa_rows = value; return 0; }
  if (key && strcmp(key, "sd_split") == 0) { cs::g_sd_split = value; return 0; }
  if (key && strcmp(key, "cap32") == 0) { cs::g_cap32 = value ? 1 : 0; return 0; }
  if (key && strcmp(key, "cap32_limit") == 0) { cs::g_cap_limit = (value > 0 && value < 200) ? value : 32; return 0; }
  cs::set_error("cs_set_tuning: unknown key");
  return CS_E_ARG;
}

int cs_extract_launches_per_image(int numOctaves, int scaleUp)
{
  if (legacy_mode())   // lowpass + (numOctaves-1) scaledown + detect + describe (+ scaleup + rescale)
    return 1 + (numOctaves - 1) + 1 + 1 + (scaleUp ? 2 : 0);
  // level-0/1 kernel + ScaleDown chain (3 levels per launch) + detect + cap fix-up + describe (+ scaleup + rescale);
  // a batch of n >= 2 images costs one launch more for the whole batch (level 1 -> 2 by the tiled ScaleDown kernel)
  return 1 + (numOctaves > 2 ? (numOctaves - 2 + 2) / 3 : 0) + 1 + (cs::g_cap32 == 0 ? 0 : 1) + 1 + (scaleUp ? 2 : 0);
}

int cs_init(int device)
{
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error("InitCuda: no CUDA device available (%s); cudasift_b200 has no CPU fallback",
              e == cudaSuccess ? "count is 0" : cudaGetErrorString(e));
    return CS_E_NODEV;
  }
  if (device < 0) device = 0;
  if (device > n - 1) device = n - 1;                      // cudaSiftH.cu:27
  CS_CUDA(cudaSetDevice(device));
  if (verbose()) {
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, device);
    printf("Device Number: %d\n  Device name: %s\n", device, prop.name);
  }
  int err = 0;
  if (!current_ctx(&err)) return err;
  return device;
}

void *cs_device_alloc(size_t bytes)
{
  void *p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes ? bytes : 1);
  if (e != cudaSuccess) { set_error("cudaMalloc(%zu): %s", bytes, cudaGetErrorString(e)); return nullptr; }
  return p;
}
int cs_device_free(void *p) { if (p) CS_CUDA(cudaFree(p)); return 0; }
int cs_memcpy_h2d(void *d, const void *h, size_t n) { CS_CUDA(cudaMemcpy(d, h, n, cudaMemcpyHostToDevice)); return 0; }
int cs_memcpy_d2h(void *h, const void *d, size_t n) { CS_CUDA(cudaMemcpy(h, d, n, cudaMemcpyDeviceToHost)); return 0; }
int cs_memset_d(void *d, int v, size_t n) { CS_CUDA(cudaMemset(d, v, n)); return 0; }
void *cs_host_alloc_pinned(size_t bytes)
{
  void *p = nullptr;
  cudaError_t e = cudaMallocHost(&p, bytes ? bytes : 1);
  if (e != cudaSuccess) { set_error("cudaMallocHost(%zu): %s", bytes, cudaGetErrorString(e)); return nullptr; }
  return p;
}
int cs_host_free_pinned(void *p) { if (p) CS_CUDA(cudaFreeHost(p)); return 0; }
int cs_device_sync(void) { CS_CUDA(cudaDeviceSynchronize()); return 0; }

size_t cs_temp_floats(int w, int h, int numOctaves, int scaleUp) { return temp_floats(w, h, numOctaves, scaleUp != 0); }

float *cs_alloc_temp(int w, int h, int numOctaves, int scaleUp)
{
  size_t fl = temp_floats(w, h, numOctaves, scaleUp != 0);
  float *p = nullptr;
  cudaError_t e = cudaMalloc((void **)&p, fl * sizeof(float));
  if (e != cudaSuccess) { set_error("AllocSiftTempMemory: cudaMalloc(%zu floats): %s", fl, cudaGetErrorString(e)); return nullptr; }
  return p;
}

int cs_free_temp(float *d_tmp)
{
  if (!d_tmp) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (c) { cudaStreamSynchronize(c->stream); c->drop_pipes(d_tmp, false); }
  CS_CUDA(cudaFree(d_tmp));
  return 0;
}

int cs_extract(const float *d_img, int w, int h, int pitch, int numOctaves, double initBlur, float thresh,
               float lowestScale, int scaleUp, float *d_tmp, void *d_pts, void *h_pts, int maxPts)
{
  return extract_sync(d_img, w, h, pitch, numOctaves, initBlur, thresh, lowestScale, scaleUp != 0, d_tmp,
                      (SiftPoint *)d_pts, (SiftPoint *)h_pts, maxPts, NULL);
}

int cs_extract_host(const float *h_img, int w, int h, int numOctaves, double initBlur, float thresh,
                    float lowestScale, int scaleUp, void *h_pts, int maxPts)
{
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  int pitch = ialignup(w, 128);
  void *d_img = nullptr, *d_pts = nullptr;
  int r;
  if ((r = c->get_scratch(0, (size_t)pitch * h * sizeof(float), &d_img)) < 0) return r;
  if ((r = c->get_scratch(1, (size_t)maxPts * sizeof(SiftPoint), &d_pts)) < 0) return r;
  CS_CUDA(cudaMemcpy2DAsync(d_img, (size_t)pitch * sizeof(float), h_img, (size_t)w * sizeof(float),
                            (size_t)w * sizeof(float), h, cudaMemcpyHostToDevice, c->stream));
  return extract_sync((const float *)d_img, w, h, pitch, numOctaves, initBlur, thresh, lowestScale, scaleUp != 0,
                      nullptr, (SiftPoint *)d_pts, (SiftPoint *)h_pts, maxPts, NULL);
}

int cs_match(void *d_s1, int n1, void *d_s2, int n2, void *h_s1, int mode, double *ms)
{
  return match_sync((SiftPoint *)d_s1, n1, (SiftPoint *)d_s2, n2, (SiftPoint *)h_s1, mode, ms);
}

int cs_match_host(void *h_s1, int n1, const void *h_s2, int n2, int mode, double *ms)
{
  int err = 0;
  if (ms) *ms = 0;
  if (n1 <= 0 || n2 <= 0) return 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  void *d1 = nullptr, *d2 = nullptr;
  int r;
  if ((r = c->get_scratch(2, (size_t)n1 * sizeof(SiftPoint), &d1)) < 0) return r;
  if ((r = c->get_scratch(3, (size_t)n2 * sizeof(SiftPoint), &d2)) < 0) return r;
  CS_CUDA(cudaMemcpyAsync(d1, h_s1, (size_t)n1 * sizeof(SiftPoint), cudaMemcpyHostToDevice, c->stream));
  CS_CUDA(cudaMemcpyAsync(d2, h_s2, (size_t)n2 * sizeof(SiftPoint), cudaMemcpyHostToDevice, c->stream));
  return match_sync((SiftPoint *)d1, n1, (SiftPoint *)d2, n2, (SiftPoint *)h_s1, mode, ms);
}

int cs_match_stats(unsigned long long out[4])
{
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  for (int i = 0; i < 4; i++) out[i] = c->matchStats[i];
  return 0;
}

// ---- stage-level entry points ----
int cs_lowpass(const float *d_src, float *d_dst, int w, int h, int pitch, float sigma)
{
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  Taps9 t; lowpass_taps(sigma, t.k);
  int r = launch_lowpass(d_src, pitch, d_dst, pitch, w, h, t, c->stream);
  if (r < 0) return r;
  CS_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

int cs_scaledown(const float *d_src, float *d_dst, int w, int h, int pitch, int newpitch)
{
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  Taps5 t; scaledown_taps(0.5f, t.k);
  int r = launch_scaledown(d_src, d_dst, w, h, pitch, newpitch, t, c->stream);
  if (r < 0) return r;
  CS_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

int cs_scaleup(const float *d_src, float *d_dst, int w, int h, int pitch, int newpitch)
{
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  int r = launch_scaleup(d_src, d_dst, w, h, pitch, newpitch, c->stream);
  if (r < 0) return r;
  CS_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

int cs_laplace_taps(int numOctaves, float initBlur, float *h_kernel)
{
  if (numOctaves < 1 || numOctaves > 7 || !h_kernel) { set_error("cs_laplace_taps: bad arguments"); return CS_E_ARG; }
  laplace_taps(numOctaves, initBlur, h_kernel);
  return 0;
}

int cs_dog_planes(const float *d_base, float *d_dog, int w, int h, int pitch, int numOctaves, int octave)
{
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if (numOctaves < 1 || numOctaves > 7 || octave < 1 || octave > numOctaves) { set_error("cs_dog_planes: bad octave"); return CS_E_ARG; }
  static float taps[8 * 12 * 16];
  memset(taps, 0, sizeof(taps));
  laplace_taps(numOctaves, 0.0f, taps);
  LaplaceTaps lt;
  for (int s = 0; s < CS_LAPLACE_S; s++)
    for (int j = 0; j < 5; j++) lt.set(s, j, taps[octave * 12 * 16 + 16 * s + j]);
  int r = launch_dog_planes(d_base, d_dog, w, h, pitch, lt, c->stream);
  if (r < 0) return r;
  CS_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

int cs_tex_probe(const float *d_img, int w, int h, int pitch, const float *d_xs, const float *d_ys, int n, float *d_out)
{
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  cudaTextureObject_t tex = 0;
  int r = make_texture(&tex, d_img, w, h, pitch);
  if (r < 0) return r;
  r = launch_tex_probe(tex, d_xs, d_ys, n, d_out, c->stream);
  cudaStreamSynchronize(c->stream);
  cudaDestroyTextureObject(tex);
  return r;
}

// ---- pipelined extractor ----
struct cs_extractor {
  int w, h, numOctaves, maxPts, scaleUp, pitch, B;
  cudaStream_t stream;
  bool legacy;
  Pipeline pipe;         // legacy per-image kernels (B == 1)
  Pipeline2 pipe2;       // batched TMA pipeline
  float *d_img;          // B staging images
  SiftPoint *d_pts;      // B x maxPts records (ranked: the output slots)
  int maxCand;           // ranked extractors: candidate records per image (0: plain extractor)
  SiftPoint *d_cand;     // ranked: B x maxCand records, written by the pipeline as d_pts is for a plain extractor
  unsigned int *d_rank;  // ranked: B x rank_scratch_words(maxCand)
  float *h_img;          // pinned, B x w x h
  uint8_t *d_u8;         // device staging for 8-bit uploads (lazily allocated)
  SiftPoint *h_pts;      // pinned, B x maxPts
  unsigned int *h_counters;   // pinned, B x CS_CNT_STRIDE
  bool hostResults;
  int lastN;
  int lastCounts[CS_MAX_BATCH];
  int lastCand[CS_MAX_BATCH];   // records found per image (ranked: in the candidate area)
  // CUDA graph of one steady-state submit (memset + kernels + count D2H).  Per image only the input pointer
  // changes: legacy = first parameter of the LowPass node, batched = the tensor maps in the parameters of the
  // first pyramid kernel; both are patched with cudaGraphExecKernelNodeSetParams.
  cudaGraphExec_t gexec;
  cudaGraph_t graph;
  cudaGraphNode_t gnode;
  cudaKernelNodeParams gparams;
  void *gargs[16];
  const float *gsrc;
  PyrAParams gpa;
  int gn, gpitch, glaunches;
  double gblur;
  float gthresh, glowest;
  int submits;
};


static void extractor_drop_graph(cs_extractor *ex)
{
  if (ex->gexec) cudaGraphExecDestroy(ex->gexec);
  if (ex->graph) cudaGraphDestroy(ex->graph);
  ex->gexec = nullptr; ex->graph = nullptr;
}

static int extractor_enqueue(cs_extractor *ex, int n, const float *const *d_imgs, int pitch, double initBlur, float thresh,
                             float lowestScale, cudaEvent_t *ev, PyrAParams *paOut)
{
  int r;
  if (ex->legacy) {
    r = ex->pipe.enqueue(d_imgs[0], pitch, initBlur, thresh, lowestScale, ex->d_pts, ex->maxPts, ex->stream, ev);
    if (r < 0) return r;
    CS_CUDA(cudaMemcpyAsync(ex->h_counters, ex->pipe.d_counters, 2 * sizeof(unsigned int), cudaMemcpyDeviceToHost, ex->stream));
  } else {
    if (ex->maxCand > 0) {
      RankParams rp;
      memset(&rp, 0, sizeof(rp));
      rp.out = ex->d_pts; rp.outStride = ex->maxPts; rp.maxOut = ex->maxPts; rp.scratch = ex->d_rank;
      r = ex->pipe2.enqueue(n, d_imgs, pitch, initBlur, thresh, lowestScale, ex->d_cand, ex->maxCand, ex->maxCand, ex->stream,
                            ev, paOut, &rp);
    } else {
      r = ex->pipe2.enqueue(n, d_imgs, pitch, initBlur, thresh, lowestScale, ex->d_pts, ex->maxPts, ex->maxPts, ex->stream, ev, paOut);
    }
    if (r < 0) return r;
    CS_CUDA(cudaMemcpyAsync(ex->h_counters, ex->pipe2.d_state, (size_t)n * CS_CNT_STRIDE * sizeof(unsigned int),
                            cudaMemcpyDeviceToHost, ex->stream));
  }
  return 0;
}

// Capture one submit into a graph.  Leaves ex->gexec == NULL if anything is unsupported; the caller then
// launches directly.
static int extractor_capture(cs_extractor *ex, int n, const float *const *d_imgs, int pitch, double initBlur, float thresh,
                             float lowestScale)
{
  if (ex->scaleUp) return 0;
  if (getenv("CUDASIFT_NO_GRAPH")) return 0;
  cudaGraph_t g = nullptr;
  if (cudaStreamBeginCapture(ex->stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { cudaGetLastError(); return 0; }
  const unsigned long long l0 = cs::g_launches;
  int r = extractor_enqueue(ex, n, d_imgs, pitch, initBlur, thresh, lowestScale, nullptr, &ex->gpa);
  ex->glaunches = (int)(cs::g_launches - l0);
  cs::g_launches = l0;                                   // captured, not launched
  cudaError_t e2 = cudaStreamEndCapture(ex->stream, &g);
  if (r < 0 || e2 != cudaSuccess || !g) { cudaGetLastError(); if (g) cudaGraphDestroy(g); return 0; }
  size_t nn = 0;
  cudaGraphGetNodes(g, nullptr, &nn);
  std::vector<cudaGraphNode_t> nodes(nn);
  cudaGraphGetNodes(g, nodes.data(), &nn);
  bool found = false;
  for (size_t i = 0; i < nn && !found; i++) {
    cudaGraphNodeType t;
    if (cudaGraphNodeGetType(nodes[i], &t) != cudaSuccess || t != cudaGraphNodeTypeKernel) continue;
    cudaKernelNodeParams kp;
    if (cudaGraphKernelNodeGetParams(nodes[i], &kp) != cudaSuccess || !kp.kernelParams) continue;
    if (ex->legacy) {   // the kernel node that reads d_img (first kernel parameter == d_img): lowpass_kernel, 7 parameters
      if (*reinterpret_cast<const float *const *>(kp.kernelParams[0]) == d_imgs[0] && kp.blockDim.x == 256) {
        ex->gnode = nodes[i]; ex->gparams = kp;
        for (int a = 0; a < 7; a++) ex->gargs[a] = kp.kernelParams[a];
        found = true;
      }
    } else if (kp.func == cs::pyr_a_func()) {
      ex->gnode = nodes[i]; ex->gparams = kp;
      found = true;
    }
  }
  cudaGraphExec_t ge = nullptr;
  if (!found || cudaGraphInstantiate(&ge, g, 0) != cudaSuccess) { cudaGetLastError(); cudaGraphDestroy(g); return 0; }
  ex->graph = g; ex->gexec = ge;
  ex->gsrc = d_imgs[0]; ex->gn = n; ex->gpitch = pitch; ex->gblur = initBlur; ex->gthresh = thresh; ex->glowest = lowestScale;
  return 0;
}

static cs_extractor *extractor_create(int w, int h, int numOctaves, int maxPts, int scaleUp, int batch, int maxCand)
{
  if (batch < 1 || batch > CS_MAX_BATCH) { set_error("cs_extractor_create_batch: batch %d out of range (1..%d)", batch, CS_MAX_BATCH); return nullptr; }
  cs_extractor *ex = new cs_extractor();
  memset((void *)ex, 0, sizeof(*ex));
  new (&ex->pipe) Pipeline();
  new (&ex->pipe2) Pipeline2();
  ex->w = w; ex->h = h; ex->numOctaves = numOctaves; ex->maxPts = maxPts; ex->scaleUp = scaleUp; ex->B = batch;
  ex->pitch = ialignup(w, 128);
  ex->legacy = legacy_mode();
  if (ex->legacy && batch != 1) { set_error("the legacy pipeline takes one image at a time"); delete ex; return nullptr; }
  bool ok = cudaStreamCreateWithFlags(&ex->stream, cudaStreamNonBlocking) == cudaSuccess;
  if (ex->legacy) ok = ok && ex->pipe.init(w, h, numOctaves, scaleUp != 0, nullptr) == 0;
  else ok = ok && ex->pipe2.init(w, h, numOctaves, scaleUp != 0, batch, nullptr) == 0;
  ok = ok && cudaMalloc((void **)&ex->d_img, (size_t)batch * ex->pitch * h * sizeof(float)) == cudaSuccess;
  ok = ok && cudaMalloc((void **)&ex->d_pts, (size_t)batch * maxPts * sizeof(SiftPoint)) == cudaSuccess;
  // the pipeline leaves some fields of a record unwritten (score, match*, empty[1..2]): make them zero, not stale memory
  ok = ok && cudaMemset(ex->d_pts, 0, (size_t)batch * maxPts * sizeof(SiftPoint)) == cudaSuccess;
  if (maxCand > 0) {
    ex->maxCand = maxCand;
    ok = ok && cudaMalloc((void **)&ex->d_cand, (size_t)batch * maxCand * sizeof(SiftPoint)) == cudaSuccess;
    ok = ok && cudaMemset(ex->d_cand, 0, (size_t)batch * maxCand * sizeof(SiftPoint)) == cudaSuccess;
    ok = ok && cudaMalloc((void **)&ex->d_rank, (size_t)batch * rank_scratch_words(maxCand) * sizeof(unsigned int)) == cudaSuccess;
  }
  ok = ok && cudaMallocHost((void **)&ex->h_img, (size_t)batch * w * h * sizeof(float)) == cudaSuccess;
  ok = ok && cudaMallocHost((void **)&ex->h_pts, (size_t)batch * maxPts * sizeof(SiftPoint)) == cudaSuccess;
  ok = ok && cudaMallocHost((void **)&ex->h_counters, (size_t)batch * CS_CNT_STRIDE * sizeof(unsigned int)) == cudaSuccess;
  if (!ok) {
    if (!cs::g_err[0]) set_error("cs_extractor_create: allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
    cs_extractor_destroy(ex);
    return nullptr;
  }
  return ex;
}

cs_extractor *cs_extractor_create_batch(int w, int h, int numOctaves, int maxPts, int scaleUp, int batch)
{
  return extractor_create(w, h, numOctaves, maxPts, scaleUp, batch, 0);
}

// Argument checks come before any CUDA call (they hold on a machine without a device).
cs_extractor *cs_extractor_create_ranked(int w, int h, int numOctaves, int maxPts, int scaleUp, int batch, int maxCandidates)
{
  if (maxPts < 1 || maxCandidates < maxPts || maxCandidates > CS_RANK_MAX_IN) {
    set_error("cs_extractor_create_ranked: invalid argument (CS_E_ARG): need 1 <= maxPts (%d) <= maxCandidates (%d) <= %d",
              maxPts, maxCandidates, CS_RANK_MAX_IN);
    return nullptr;
  }
  if (legacy_mode()) {
    set_error("cs_extractor_create_ranked: invalid argument (CS_E_ARG): ranking runs on the batched pipeline only (legacy is set)");
    return nullptr;
  }
  return extractor_create(w, h, numOctaves, maxPts, scaleUp, batch, maxCandidates);
}

cs_extractor *cs_extractor_create(int w, int h, int numOctaves, int maxPts, int scaleUp)
{
  return cs_extractor_create_batch(w, h, numOctaves, maxPts, scaleUp, 1);
}

int cs_extractor_destroy(cs_extractor *ex)
{
  if (!ex) return 0;
  if (ex->stream) cudaStreamSynchronize(ex->stream);
  extractor_drop_graph(ex);
  ex->pipe.destroy();
  ex->pipe2.destroy();
  if (ex->d_img) cudaFree(ex->d_img);
  if (ex->d_u8) cudaFree(ex->d_u8);
  if (ex->d_pts) cudaFree(ex->d_pts);
  if (ex->d_cand) cudaFree(ex->d_cand);
  if (ex->d_rank) cudaFree(ex->d_rank);
  if (ex->h_img) cudaFreeHost(ex->h_img);
  if (ex->h_pts) cudaFreeHost(ex->h_pts);
  if (ex->h_counters) cudaFreeHost(ex->h_counters);
  if (ex->stream) cudaStreamDestroy(ex->stream);
  delete ex;
  return 0;
}

int cs_extractor_submit_device_batch(cs_extractor *ex, int n, const float *const *d_imgs, int pitch, double initBlur,
                                     float thresh, float lowestScale)
{
  if (n < 1 || n > ex->B || !d_imgs) { set_error("cs_extractor_submit: batch of %d on an extractor built for %d", n, ex->B); return CS_E_ARG; }
  ex->hostResults = false;
  ex->lastN = n;
  ex->submits++;
  if (!ex->legacy)
    for (int i = 0; i < n; i++)
      if (!tensor_map_compatible(d_imgs[i], pitch)) {
        set_error("cs_extractor_submit: image %d (%p, pitch %d) must be 16-byte aligned with a pitch that is a multiple of 4 "
                  "floats (or use CUDASIFT_LEGACY=1)", i, (const void *)d_imgs[i], pitch);
        return CS_E_ARG;
      }
  if (ex->gexec && (n != ex->gn || pitch != ex->gpitch || initBlur != ex->gblur || thresh != ex->gthresh || lowestScale != ex->glowest)) {
    extractor_drop_graph(ex);                                           // parameters changed: re-capture
    ex->submits = 2;
  }
  if (!ex->gexec && ex->submits == 2) extractor_capture(ex, n, d_imgs, pitch, initBlur, thresh, lowestScale);
  if (ex->gexec) {
    if (ex->legacy) {
      if (d_imgs[0] != ex->gsrc) {
        const float *src = d_imgs[0];
        cudaKernelNodeParams kp = ex->gparams;
        void *args[7];
        for (int a = 0; a < 7; a++) args[a] = ex->gargs[a];
        args[0] = (void *)&src;
        kp.kernelParams = args;
        CS_CUDA(cudaGraphExecKernelNodeSetParams(ex->gexec, ex->gnode, &kp));
        ex->gsrc = d_imgs[0];
      }
    } else {
      int r = ex->pipe2.fill_pyr_a(ex->gpa, n, d_imgs, pitch, initBlur);
      if (r < 0) return r;
      cudaKernelNodeParams kp = ex->gparams;
      void *args[1] = {(void *)&ex->gpa};
      kp.kernelParams = args;
      CS_CUDA(cudaGraphExecKernelNodeSetParams(ex->gexec, ex->gnode, &kp));
    }
    CS_CUDA(cudaGraphLaunch(ex->gexec, ex->stream));
    count_launch(ex->glaunches);
    return 0;
  }
  return extractor_enqueue(ex, n, d_imgs, pitch, initBlur, thresh, lowestScale, nullptr, nullptr);
}

int cs_extractor_submit_device(cs_extractor *ex, const float *d_img, int pitch, double initBlur, float thresh,
                               float lowestScale)
{
  return cs_extractor_submit_device_batch(ex, 1, &d_img, pitch, initBlur, thresh, lowestScale);
}

int cs_extractor_submit_host_batch(cs_extractor *ex, int n, const float *const *h_imgs, double initBlur, float thresh,
                                   float lowestScale)
{
  if (n < 1 || n > ex->B || !h_imgs) { set_error("cs_extractor_submit_host: batch of %d on an extractor built for %d", n, ex->B); return CS_E_ARG; }
  const float *dptr[CS_MAX_BATCH];
  for (int i = 0; i < n; i++) {
    float *d = ex->d_img + (size_t)i * ex->pitch * ex->h;
    CS_CUDA(cudaMemcpy2DAsync(d, (size_t)ex->pitch * sizeof(float), h_imgs[i], (size_t)ex->w * sizeof(float),
                              (size_t)ex->w * sizeof(float), ex->h, cudaMemcpyHostToDevice, ex->stream));
    dptr[i] = d;
  }
  int r = cs_extractor_submit_device_batch(ex, n, dptr, ex->pitch, initBlur, thresh, lowestScale);
  ex->hostResults = true;
  return r;
}

int cs_extractor_submit_host(cs_extractor *ex, const float *h_img, double initBlur, float thresh, float lowestScale)
{
  return cs_extractor_submit_host_batch(ex, 1, &h_img, initBlur, thresh, lowestScale);
}

int cs_extractor_submit_host_u8(cs_extractor *ex, const unsigned char *h_img, double initBlur, float thresh,
                                float lowestScale)
{
  const int p8 = ialignup(ex->w, 128);
  if (!ex->d_u8) CS_CUDA(cudaMalloc((void **)&ex->d_u8, (size_t)p8 * ex->h));
  CS_CUDA(cudaMemcpy2DAsync(ex->d_u8, p8, h_img, ex->w, ex->w, ex->h, cudaMemcpyHostToDevice, ex->stream));
  int r = launch_u8_to_float(ex->d_u8, p8, ex->d_img, ex->pitch, ex->w, ex->h, ex->stream);
  if (r < 0) return r;
  r = cs_extractor_submit_device(ex, ex->d_img, ex->pitch, initBlur, thresh, lowestScale);
  ex->hostResults = true;
  return r;
}

int cs_extractor_wait_batch(cs_extractor *ex, int *counts)
{
  CS_CUDA(cudaStreamSynchronize(ex->stream));
  const int n = ex->lastN > 0 ? ex->lastN : 1;
  int total = 0;
  bool copies = false;
  for (int i = 0; i < n; i++) {
    const unsigned int *hc = ex->h_counters + (size_t)i * CS_CNT_STRIDE;
    int c;
    if (ex->maxCand > 0) {                       // ranked: [2] = records in the output slot
      c = (int)(hc[2] < (unsigned)ex->maxPts ? hc[2] : (unsigned)ex->maxPts);
      ex->lastCand[i] = count_from_counters(hc, ex->maxCand);
    } else {
      c = count_from_counters(hc, ex->maxPts);
      ex->lastCand[i] = c;
    }
    ex->lastCounts[i] = c;
    if (counts) counts[i] = c;
    total += c;
    if (ex->hostResults && c > 0) {
      CS_CUDA(cudaMemcpyAsync(ex->h_pts + (size_t)i * ex->maxPts, ex->d_pts + (size_t)i * ex->maxPts, sizeof(SiftPoint) * (size_t)c,
                              cudaMemcpyDeviceToHost, ex->stream));
      copies = true;
    }
  }
  if (copies) CS_CUDA(cudaStreamSynchronize(ex->stream));
  return total;
}

int cs_extractor_wait(cs_extractor *ex) { return cs_extractor_wait_batch(ex, nullptr); }

int cs_extractor_profile_batch(cs_extractor *ex, int n, const float *const *d_imgs, int pitch, double initBlur, float thresh,
                               float lowestScale, float out_ms[5])
{
  if (n < 1 || n > ex->B) { set_error("cs_extractor_profile: bad batch"); return CS_E_ARG; }
  const int ne = ex->maxCand > 0 ? 6 : 5;       // ranked: one more event, after the ranking stage
  cudaEvent_t ev[6];
  for (int i = 0; i < ne; i++) CS_CUDA(cudaEventCreate(&ev[i]));
  ex->lastN = n;
  int r = extractor_enqueue(ex, n, d_imgs, pitch, initBlur, thresh, lowestScale, ev, nullptr);
  if (r < 0) { for (int i = 0; i < ne; i++) cudaEventDestroy(ev[i]); return r; }
  CS_CUDA(cudaStreamSynchronize(ex->stream));
  for (int i = 0; i < 4; i++) cudaEventElapsedTime(&out_ms[i], ev[i], ev[i + 1]);
  cudaEventElapsedTime(&out_ms[4], ev[0], ev[ne - 1]);
  for (int i = 0; i < ne; i++) cudaEventDestroy(ev[i]);
  ex->hostResults = false;
  return cs_extractor_wait_batch(ex, nullptr);
}

int cs_extractor_profile(cs_extractor *ex, const float *d_img, int pitch, double initBlur, float thresh,
                         float lowestScale, float out_ms[5])
{
  return cs_extractor_profile_batch(ex, 1, &d_img, pitch, initBlur, thresh, lowestScale, out_ms);
}

// One pyramid level of image slot `slot` after the last submit (parity tests): copies lw x lh floats (packed)
// to h_out; returns the level's width | height << 16, or a negative code.
int cs_extractor_read_level(cs_extractor *ex, int slot, int level, float *h_out)
{
  CS_CUDA(cudaStreamSynchronize(ex->stream));
  const float *src; int lw, lh, lp;
  if (ex->legacy) {
    if (slot != 0 || level < 0 || level >= ex->pipe.numLevels) { set_error("cs_extractor_read_level: bad level"); return CS_E_ARG; }
    src = ex->pipe.lev[level]; lw = ex->pipe.lw[level]; lh = ex->pipe.lh[level]; lp = ex->pipe.lp[level];
  } else {
    if (slot < 0 || slot >= ex->B || level < 0 || level >= ex->pipe2.numLevels) { set_error("cs_extractor_read_level: bad level"); return CS_E_ARG; }
    src = ex->pipe2.level(slot, level); lw = ex->pipe2.lw[level]; lh = ex->pipe2.lh[level]; lp = ex->pipe2.lp[level];
  }
  if (h_out)
    CS_CUDA(cudaMemcpy2D(h_out, (size_t)lw * sizeof(float), src, (size_t)lp * sizeof(float), (size_t)lw * sizeof(float), lh,
                         cudaMemcpyDeviceToHost));
  return lw | (lh << 16);
}

int cs_extractor_count(cs_extractor *ex, int slot) { return (slot >= 0 && slot < CS_MAX_BATCH) ? ex->lastCounts[slot] : 0; }
int cs_extractor_candidates(cs_extractor *ex, int slot) { return (slot >= 0 && slot < CS_MAX_BATCH) ? ex->lastCand[slot] : 0; }

int cs_rank_records(const void *d_in, int n, void *d_out, int maxOut)
{
  if (n < 0 || n > CS_RANK_MAX_IN || maxOut < 1 || (n > 0 && (!d_in || !d_out)) ||
      ((reinterpret_cast<uintptr_t>(d_in) | reinterpret_cast<uintptr_t>(d_out)) & 15) != 0) {
    set_error("cs_rank_records: need 0 <= n (%d) <= %d, maxOut (%d) >= 1 and 16-byte aligned record arrays", n, CS_RANK_MAX_IN, maxOut);
    return CS_E_ARG;
  }
  if (n == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  void *buf = nullptr;
  const size_t words = CS_CNT_STRIDE + rank_scratch_words(n);   // counters | scratch
  int r = c->get_scratch(4, words * sizeof(unsigned int), &buf);
  if (r < 0) return r;
  unsigned int *cnt = (unsigned int *)buf;
  const unsigned int init[CS_CNT_STRIDE] = {(unsigned)n, (unsigned)n, 0u, 0u};
  CS_CUDA(cudaMemcpyAsync(cnt, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
  RankParams rp;
  memset(&rp, 0, sizeof(rp));
  rp.in = (const SiftPoint *)d_in; rp.maxIn = n;
  rp.out = (SiftPoint *)d_out; rp.maxOut = maxOut;
  rp.counters = cnt; rp.scratch = cnt + CS_CNT_STRIDE;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if ((r = launch_rank(rp, 1, sms, c->stream)) < 0) return r;
  CS_CUDA(cudaMemcpyAsync(c->h_counters, cnt, CS_CNT_STRIDE * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
  CS_CUDA(cudaStreamSynchronize(c->stream));
  return (int)c->h_counters[2];
}

// ---- device timers (CUDA events on the extractor's own stream) ----
void *cs_event_create(void)
{
  cudaEvent_t e = nullptr;
  if (cudaEventCreate(&e) != cudaSuccess) { set_error("cudaEventCreate failed"); return nullptr; }
  return (void *)e;
}
int cs_event_destroy(void *ev) { if (ev) cudaEventDestroy((cudaEvent_t)ev); return 0; }
int cs_event_record(void *ev, cs_extractor *ex)
{
  CS_CUDA(cudaEventRecord((cudaEvent_t)ev, ex ? ex->stream : (cudaStream_t)0));
  return 0;
}
double cs_event_elapsed_ms(void *a, void *b)
{
  float ms = 0.0f;
  cudaEventSynchronize((cudaEvent_t)b);
  if (cudaEventElapsedTime(&ms, (cudaEvent_t)a, (cudaEvent_t)b) != cudaSuccess) return -1.0;
  return ms;
}

void *cs_extractor_device_points(cs_extractor *ex) { return ex->d_pts; }
void *cs_extractor_host_points(cs_extractor *ex) { return ex->h_pts; }
float *cs_extractor_host_image(cs_extractor *ex) { return ex->h_img; }
void *cs_extractor_device_points_at(cs_extractor *ex, int slot) { return ex->d_pts + (size_t)slot * ex->maxPts; }
void *cs_extractor_host_points_at(cs_extractor *ex, int slot) { return ex->h_pts + (size_t)slot * ex->maxPts; }
float *cs_extractor_host_image_at(cs_extractor *ex, int slot) { return ex->h_img + (size_t)slot * ex->w * ex->h; }
int cs_max_batch(void) { return CS_MAX_BATCH; }

// Host logic only (no device needed): the detector's work list for `n` images of width x height; every item is
// 4 ints {level | image << 8, x0, first tested row, rows per stream}.  Returns the number of items.
int cs_detector_items(int width, int height, int numOctaves, int scaleUp, int n, int hs, unsigned int *out, int capItems)
{
  if (width < 1 || height < 1 || numOctaves < 1 || numOctaves > 7 || n < 1 || hs < 1) { set_error("cs_detector_items: bad arguments"); return CS_E_ARG; }
  int lw[CS_MAX_LEVELS], lh[CS_MAX_LEVELS], nl = numOctaves;
  lw[0] = width * (scaleUp ? 2 : 1); lh[0] = height * (scaleUp ? 2 : 1);
  for (int i = 1; i < numOctaves; i++) { lw[i] = lw[i - 1] / 2; lh[i] = lh[i - 1] / 2; if (lw[i] < 1 || lh[i] < 1) { nl = i; break; } }
  std::vector<uint4> v;
  cs::build_detector_items(lw, lh, nl, n, hs, v);
  for (size_t i = 0; i < v.size() && (int)i < capItems; i++) {
    out[4 * i] = v[i].x; out[4 * i + 1] = v[i].y; out[4 * i + 2] = v[i].z; out[4 * i + 3] = v[i].w;
  }
  return (int)v.size();
}

}  // extern "C"
