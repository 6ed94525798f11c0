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
#include "args.h"
#include "pipeline2.h"

#include <algorithm>
#include <cmath>
#include <cstddef>
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

static inline int count_from_counters(const unsigned int *c, int maxPts)
{
  unsigned int a = c[0] < (unsigned)maxPts ? c[0] : (unsigned)maxPts;
  unsigned int b = c[1] < (unsigned)maxPts ? c[1] : (unsigned)maxPts;
  return (int)(a > b ? a : b);
}

// ------------------------------------------------------------------------------ device ctx
int DeviceCtx::ensure(int d)
{
  if (dev == d && stream) return 0;
  dev = d;
  CS_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, d));
  // the stream last: a context that has one has every pinned word
  if (!h_counters) CS_CUDA(cudaMallocHost((void **)&h_counters, 4 * sizeof(unsigned int)));
  if (!h_tcFlags) CS_CUDA(cudaMallocHost((void **)&h_tcFlags, 16 * sizeof(unsigned int)));
  if (!h_pairTotal) CS_CUDA(cudaMallocHost((void **)&h_pairTotal, sizeof(unsigned int)));
  CS_CUDA(cudaStreamCreate(&stream));
  return 0;
}
Pipeline *DeviceCtx::get_pipe(int w, int h, int oct, bool up, float *arena, int *err)
{
  PipeKey k{w, h, oct, up ? 1 : 0, arena};
  auto it = pipes.find(k);
  if (it != pipes.end()) return it->second;
  if (!arena && pipes.size() > 8) drop_pipes(nullptr, true);   // bound the internal-arena cache
  Pipeline *p = new Pipeline();
  int r = p->init(w, h, oct, up, 1, arena);
  if (r < 0) { p->destroy(); delete p; *err = r; return nullptr; }
  pipes[k] = p;
  return p;
}
void DeviceCtx::drop_pipes(float *arena, bool internalOnly)
{
  for (auto it = pipes.begin(); it != pipes.end();) {
    bool hit = internalOnly ? it->second->ownArena : (it->first.arena == arena);
    if (hit) { it->second->destroy(); delete it->second; it = pipes.erase(it); }
    else ++it;
  }
}

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
  if ((err = check_level0_size("ExtractSift", w, h, scaleUp)) < 0) return err;
  if (!d_img || !d_pts || maxPts < 1) { set_error("ExtractSift: missing image or SiftData"); return CS_E_ARG; }
  if ((reinterpret_cast<uintptr_t>(d_tmp) & 15) != 0) {   // the level textures and tensor maps start in it
    set_error("ExtractSift: tempMemory %p must be 16-byte aligned", (void *)d_tmp);
    return CS_E_ARG;
  }
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  Pipeline *p = c->get_pipe(w, h, numOctaves, scaleUp, d_tmp, &err);
  if (!p) return err;
  // the round-1 kernels: asked for, or an image (or arena) TMA cannot address
  const bool round1 = legacy_mode() || !p->tma || !tensor_map_compatible(d_img, pitch);
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (msKernel) { cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventRecord(e0, c->stream); }
  int r = round1 ? p->enqueue_round1(d_img, pitch, initBlur, thresh, lowestScale, d_pts, maxPts, c->stream)
                 : p->enqueue(1, &d_img, pitch, initBlur, thresh, lowestScale, d_pts, 0, maxPts, c->stream);
  if (r < 0) { if (msKernel) { cudaEventDestroy(e0); cudaEventDestroy(e1); } return r; }
  if (msKernel) cudaEventRecord(e1, c->stream);
  CS_CUDA(cudaMemcpyAsync(c->h_counters, p->counters(0), 2 * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
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

// Runs enqueue() on c's stream between two events, then synchronizes; *ms (when given) receives the time between the
// events if all went well.  A failed synchronize is CS_E_CUDA, its message prefixed by fn.  Returns enqueue's result.
template <class Enqueue>
static int timed_sync(const char *fn, DeviceCtx *c, double *ms, Enqueue &&enqueue)
{
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0, c->stream);
  int r = enqueue();
  if (r >= 0) {
    cudaEventRecord(e1, c->stream);
    cudaError_t ce = cudaStreamSynchronize(c->stream);
    if (ce != cudaSuccess) { set_error("%s: %s", fn, cudaGetErrorString(ce)); r = CS_E_CUDA; }
  }
  if (r >= 0 && ms) { float t = 0; cudaEventElapsedTime(&t, e0, e1); *ms = t; }
  cudaEventDestroy(e0); cudaEventDestroy(e1);                              // on every path
  return r;
}

// CUDA events between the kernels, printed to stderr (warm caches, unlike ncu)
cudaEvent_t *match_timing_events()
{
  static int timing = -1;
  static cudaEvent_t tev[9];
  if (timing < 0) {
    const char *e = getenv("CUDASIFT_MATCH_TIMING");
    timing = (e && atoi(e)) ? 1 : 0;
    if (timing) for (int i = 0; i < 9; i++) cudaEventCreate(&tev[i]);
  }
  return timing ? tev : nullptr;
}

void report_stage_times(const cudaEvent_t *tev, const char *const *names, int n, const char *header, ...)
{
  cudaEventSynchronize(tev[n]);
  va_list ap;
  va_start(ap, header);
  vfprintf(stderr, header, ap);
  va_end(ap);
  fprintf(stderr, " [us]:");
  for (int i = 0; i < n; i++) {
    float ms = 0.0f;
    cudaEventElapsedTime(&ms, tev[i], tev[i + 1]);
    fprintf(stderr, " %s %.1f", names[i], ms * 1e3f);
  }
  fprintf(stderr, "\n");
}

// cs_match_stats after a finished match or knn call: the tensor path's counters (a two-way call: both directions
// summed) and the path taken
static void set_match_stats(DeviceCtx *c, bool tensor)
{
  c->matchStats[0] = c->matchStats[1] = c->matchStats[2] = 0;
  if (tensor) match_tensor_stats(*c, c->matchStats);
  c->matchStats[3] = tensor ? 2 : 1;
}

// Set 1's five match fields on the device, copied to h_s1 when given.  With mu also set 2's, as a match of set 2 against
// set 1 writes them (copied to h_s2 when given), then the cross-checked pairs; the call then returns the number of
// pairs.  fn prefixes the error messages.  *ms covers the copies to the host.
static int match_sync(const char *fn, SiftPoint *d_s1, int n1, SiftPoint *d_s2, int n2, const MutualArgs *mu, int mode,
                      SiftPoint *h_s1, SiftPoint *h_s2, double *ms)
{
  int err = 0;
  if (ms) *ms = 0.0;
  if (!n1 || !n2) return 0;                                                // matching.cu:1095-1096
  if (!d_s1 || !d_s2) return 0;                                            // matching.cu:1101-1102
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  // The tensor path: asked for (mode 2) or automatic for 256 x 256 and more.  A one-way call with fewer than 32
  // candidates runs the exact kernel inside match_tensor and reports path 2; a mutual call takes the exact path unless
  // both sets have 32 rows.
  bool tensor = (mode == 2) || (mode == 0 && match_tensor_supported() && n1 >= 256 && n2 >= 256);
  if (mu) tensor = tensor && match_tensor_supported() && n1 >= 32 && n2 >= 32;
  auto enqueue = [&]() -> int {
    int r;
    if (tensor) {
      r = match_tensor(*c, d_s1, n1, d_s2, n2, mu);
    } else {
      r = match_exact(d_s1, n1, d_s2, n2, c->stream);
      if (mu && r >= 0) r = match_exact(d_s2, n2, d_s1, n1, c->stream);
      if (mu && r >= 0) r = launch_mutual_pairs(*c, d_s1, n1, d_s2, n2, *mu);
    }
    const SiftPoint *dev[2] = {d_s1, d_s2};
    SiftPoint *host[2] = {h_s1, h_s2};
    const int cnt[2] = {n1, n2};
    for (int k = 0; k < 2 && r >= 0; k++) {                                // matching.cu:1195-1199
      if (!host[k]) continue;
      cudaError_t ce = cudaMemcpy2DAsync(&host[k][0].score, sizeof(SiftPoint), &dev[k][0].score, sizeof(SiftPoint),
                                         5 * sizeof(float), cnt[k], cudaMemcpyDeviceToHost, c->stream);
      if (ce != cudaSuccess) { set_error("%s: result copy failed: %s", fn, cudaGetErrorString(ce)); r = CS_E_CUDA; }
    }
    return r;
  };
  const int r = timed_sync(fn, c, ms, enqueue);
  if (r < 0) return r;
  set_match_stats(c, tensor);
  return mu ? (int)*c->h_pairTotal : 0;
}

// The two host sets to the context's set buffers (the caller's stream order makes them visible to the match).
static int upload_sets(DeviceCtx *c, const void *h_s1, int n1, const void *h_s2, int n2)
{
  int r;
  if ((r = c->set1.grow((size_t)n1 * sizeof(SiftPoint))) < 0) return r;
  if ((r = c->set2.grow((size_t)n2 * sizeof(SiftPoint))) < 0) return r;
  CS_CUDA(cudaMemcpyAsync(c->set1.p, h_s1, (size_t)n1 * sizeof(SiftPoint), cudaMemcpyHostToDevice, c->stream));
  CS_CUDA(cudaMemcpyAsync(c->set2.p, h_s2, (size_t)n2 * sizeof(SiftPoint), cudaMemcpyHostToDevice, c->stream));
  return 0;
}

// The shared path of the *_host entry points that return pairs: the sets uploaded, then run(d1, d2, buf) -- the device
// variant, with the context's pair buffer of `entries` int2 as buf -- and min(total, room) pairs from buf + at copied
// to h_out.  Returns run's total.
template <class Run>
static int host_pairs(DeviceCtx *c, const void *h_s1, int n1, const void *h_s2, int n2, size_t entries, size_t at,
                      int room, int *h_out, Run &&run)
{
  int r;
  if ((r = c->pairs.grow(entries * sizeof(int2))) < 0) return r;
  if ((r = upload_sets(c, h_s1, n1, h_s2, n2)) < 0) return r;
  int2 *buf = c->pairs.as<int2>();
  const int total = run(c->set1.as<SiftPoint>(), c->set2.as<SiftPoint>(), buf);
  if (total < 0) return total;
  const int k = total < room ? total : room;
  if (k > 0) CS_CUDA(cudaMemcpy(h_out, buf + at, (size_t)k * sizeof(int2), cudaMemcpyDeviceToHost));
  return total;
}

// The two nearest neighbours of set 1's rows in set 2 (idx1 / score1, [n1][2]); with idx2 also those of set 2's rows in
// set 1; with ra then the ratio-test pairs, cross-checked when idx2 is given, and the call returns their number.  The
// records are only read; both sets are non-empty.  Path rule: the tensor path when asked for (mode 2) or automatically
// for 256 x 256 and more.
static int knn_sync(const char *fn, DeviceCtx *c, const SiftPoint *d_s1, int n1, const SiftPoint *d_s2, int n2,
                    int *idx1, float *score1, int *idx2, float *score2, const RatioArgs *ra, int mode, double *ms)
{
  const bool tensor = match_tensor_supported() && (mode == 2 || (mode == 0 && n1 >= 256 && n2 >= 256));
  auto enqueue = [&]() -> int {
    int r;
    if (tensor) {
      r = match_knn_tensor(*c, d_s1, n1, d_s2, n2, idx1, score1, idx2, score2);
    } else {
      r = knn_exact(*c, d_s1, n1, d_s2, n2, idx1, score1);
      if (idx2 && r >= 0) r = knn_exact(*c, d_s2, n2, d_s1, n1, idx2, score2);
    }
    if (ra && r >= 0) r = launch_ratio_pairs(*c, idx1, score1, n1, idx2, score2, n2, *ra);
    return r;
  };
  const int r = timed_sync(fn, c, ms, enqueue);
  if (r < 0) return r;
  set_match_stats(c, tensor);
  return ra ? (int)*c->h_pairTotal : 0;
}

// The knn lists of a ratio call in the context's knnLists: set 1's rows, and with crossCheck set 2's (else null).
struct KnnLists {
  int *idx1, *idx2;
  float *sc1, *sc2;
};
static int knn_lists(DeviceCtx *c, int n1, int n2, bool crossCheck, KnnLists *l)
{
  const size_t a = ialignup(2 * n1, 64), b = crossCheck ? ialignup(2 * n2, 64) : 0;
  int r;
  if ((r = c->knnLists.grow((2 * a + 2 * b) * sizeof(int))) < 0) return r;
  l->idx1 = c->knnLists.as<int>();
  l->idx2 = crossCheck ? l->idx1 + 2 * a : nullptr;
  l->sc1 = reinterpret_cast<float *>(l->idx1 + a);
  l->sc2 = crossCheck ? reinterpret_cast<float *>(l->idx2 + b) : nullptr;
  return 0;
}

// cs_match_ratio on device sets.
static int ratio_sync(const char *fn, DeviceCtx *c, const SiftPoint *d1, int n1, const SiftPoint *d2, int n2,
                      const RatioArgs &ra, bool crossCheck, int mode, double *ms)
{
  KnnLists l;
  const int r = knn_lists(c, n1, n2, crossCheck, &l);
  if (r < 0) return r;
  return knn_sync(fn, c, d1, n1, d2, n2, l.idx1, l.sc1, l.idx2, l.sc2, &ra, mode, ms);
}

// cs_match_knn2_guided / cs_match_guided on non-empty device sets: one job of guided_enqueue over the sets {d1, d2}.
// With ra its ratio-test pairs (cross-checked with crossCheck), and the call returns their number; without ra set 1's
// lists go to idx / score.  One synchronize; the job's statistics become cs_match_guided_stats.
static int guided_sync(const char *fn, DeviceCtx *c, const void *d1, int n1, const void *d2, int n2, int model,
                       const double *model_in, float thresh, const RatioArgs *ra, bool crossCheck, int *idx,
                       float *score, double *ms)
{
  const cs_match_set sets[2] = {{d1, n1}, {d2, n2}};
  const cs_match_job job = {0, 1, ra ? reinterpret_cast<int *>(ra->pairs) : nullptr, ra ? ra->maxPairs : 0};
  const GuidedSingle single = {idx, score};
  GuidedBatchOut out = {nullptr, nullptr};
  const int r = timed_sync(fn, c, ms, [&]() {
    return guided_enqueue(*c, sets, &job, 1, &model, model_in, thresh, ra ? ra->maxRatio : 0.0f,
                          ra ? ra->maxDistance : 0.0f, crossCheck, &out, &single);
  });
  if (r < 0) return r;
  for (int k = 0; k < 4; k++) c->guidedStats[k] = out.stats[k];
  return ra ? (int)*out.total : 0;
}

static cs_verify_job verify_job(const SiftPoint *d1, int n1, const SiftPoint *d2, int n2, const int *pairs, int numPairs,
                                unsigned long long seed, int *inliers, int maxInliers)
{
  cs_verify_job j;
  j.s1 = d1; j.n1 = n1; j.s2 = d2; j.n2 = n2; j.pairs = pairs; j.numPairs = numPairs;
  j.seed = seed; j.inliers = inliers; j.maxInliers = maxInliers;
  return j;
}

// The launches of a batch (cal: per job, essential only) and one synchronize.
static int verify_batch_sync(const char *fn, DeviceCtx *c, const cs_verify_job *jobs, int numJobs, const VerifyCalib *cal,
                             int model, int numLoops, float thresh, double *ms)
{
  return timed_sync(fn, c, ms, [&] { return verify_enqueue(*c, jobs, numJobs, cal, model, numLoops, thresh, true); });
}

// The shared path of cs_verify_pairs_host and cs_verify_essential_host: the sets and the input pairs uploaded, then
// run(job) -- the single call as a job on them, its inliers after the pairs in the context's pair buffer -- and the
// inliers copied to h_inliers.  Returns run's total.
template <class Run>
static int verify_host_pairs(DeviceCtx *c, const void *h_s1, int n1, const void *h_s2, int n2, const int *h_pairs,
                             int numPairs, unsigned long long seed, int *h_inliers, int maxInliers, Run &&run)
{
  const int room = maxInliers < numPairs ? maxInliers : numPairs;     // no more inliers can exist
  // the pair buffer holds the input pairs, then room inliers
  return host_pairs(c, h_s1, n1, h_s2, n2, (size_t)numPairs + room, numPairs, room, h_inliers,
                    [&](SiftPoint *d1, SiftPoint *d2, int2 *pairs) {
                      CS_CUDA(cudaMemcpyAsync(pairs, h_pairs, (size_t)numPairs * sizeof(int2), cudaMemcpyHostToDevice,
                                              c->stream));
                      return run(verify_job(d1, n1, d2, n2, reinterpret_cast<int *>(pairs), numPairs, seed,
                                            reinterpret_cast<int *>(pairs + numPairs), room));
                    });
}

// The body of a batch entry point after its argument checks: every job's outputs zeroed (zero(p), the count and
// numStats statistics); when some job has work (work(p)), enqueue(c) and one synchronize; then the count and statistics
// of every job with work from result(c, p, q, st), job p being the q-th with work and st numStats zeros on entry.
template <class Stat, class Zero, class Work, class Enqueue, class Result>
static int batch_body(const char *fn, int numJobs, int *counts_out, Stat *stats_out, int numStats, double *ms,
                      Zero &&zero, Work &&work, Enqueue &&enqueue, Result &&result)
{
  bool any = false;
  for (int p = 0; p < numJobs; p++) {
    zero(p);
    counts_out[p] = 0;
    if (stats_out)
      for (int k = 0; k < numStats; k++) stats_out[numStats * (size_t)p + k] = 0;
    any |= work(p);
  }
  if (!any) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  int r;
  if ((r = timed_sync(fn, c, ms, [&] { return enqueue(c); })) < 0) return r;
  for (int p = 0, q = 0; p < numJobs; p++) {
    if (!work(p)) continue;
    Stat st[10] = {};
    counts_out[p] = result(c, p, q++, st);
    if (stats_out)
      for (int k = 0; k < numStats; k++) stats_out[numStats * (size_t)p + k] = st[k];
  }
  return 0;
}

// cs_verify_models / cs_verify_essential_models: steps 1-4 of one job, then its slots to the host.
static int verify_models_sync(DeviceCtx *c, const cs_verify_job &job, const VerifyCalib *cal, int model, int numLoops,
                              float thresh, double *h_models, int *h_counts, double h_norm[5])
{
  int r;
  if ((r = verify_enqueue(*c, &job, 1, cal, model, numLoops, thresh, false)) < 0) return r;
  return verify_models_to_host(*c, job, numLoops, model, cal, h_models, h_counts, h_norm);
}

static VerifyCalib verify_calib(const double K1[9], const double K2[9])
{
  VerifyCalib cal;
  for (int k = 0; k < 9; k++) { cal.K1[k] = K1[k]; cal.K2[k] = K2[k]; }
  return cal;
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
  int r = match_sync("MatchSiftData", data1.m_data, data1.numPts, data2.m_data, data2.numPts, NULL, 0, NULL, NULL, &ms);
#else
  int r = match_sync("MatchSiftData", data1.d_data, data1.numPts, data2.d_data, data2.numPts, NULL, 0, data1.h_data, NULL,
                     &ms);
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
  if (key && strcmp(key, "texture_group_bytes") == 0) { cs::g_texture_group_bytes = value; return 0; }
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
  if ((err = check_level0_size("ExtractSift", w, h, scaleUp != 0)) < 0) return err;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  int pitch = ialignup(w, 128);
  int r;
  if ((r = c->image.grow((size_t)pitch * h * sizeof(float))) < 0) return r;
  if ((r = c->points.grow((size_t)maxPts * sizeof(SiftPoint))) < 0) return r;
  CS_CUDA(cudaMemcpy2DAsync(c->image.p, (size_t)pitch * sizeof(float), h_img, (size_t)w * sizeof(float),
                            (size_t)w * sizeof(float), h, cudaMemcpyHostToDevice, c->stream));
  return extract_sync(c->image.as<const float>(), w, h, pitch, numOctaves, initBlur, thresh, lowestScale, scaleUp != 0,
                      nullptr, c->points.as<SiftPoint>(), (SiftPoint *)h_pts, maxPts, NULL);
}

int cs_match(void *d_s1, int n1, void *d_s2, int n2, void *h_s1, int mode, double *ms)
{
  return match_sync("MatchSiftData", (SiftPoint *)d_s1, n1, (SiftPoint *)d_s2, n2, nullptr, mode, (SiftPoint *)h_s1, nullptr,
                    ms);
}

int cs_match_host(void *h_s1, int n1, const void *h_s2, int n2, int mode, double *ms)
{
  int err = 0;
  if (ms) *ms = 0;
  if (n1 <= 0 || n2 <= 0) return 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  int r;
  if ((r = upload_sets(c, h_s1, n1, h_s2, n2)) < 0) return r;
  return match_sync("MatchSiftData", c->set1.as<SiftPoint>(), n1, c->set2.as<SiftPoint>(), n2, nullptr, mode,
                    (SiftPoint *)h_s1, nullptr, ms);
}

int cs_match_mutual(void *d_s1, int n1, void *d_s2, int n2, float minScore, float maxAmbiguity, int *d_pairs, int maxPairs,
                    int mode, double *ms)
{
  const char *fn = "cs_match_mutual";
  if (ms) *ms = 0.0;
  int r = mutual_args(fn, d_s1, n1, d_s2, n2, d_pairs, maxPairs, mode);
  if (r < 0) return r;
  if ((reinterpret_cast<uintptr_t>(d_pairs) & 7) != 0)                 // also when maxPairs is 0
    return arg_error(fn, "pairs must be 8-byte aligned");
  const MutualArgs mu = {minScore, maxAmbiguity, (int2 *)d_pairs, maxPairs};
  return match_sync(fn, (SiftPoint *)d_s1, n1, (SiftPoint *)d_s2, n2, &mu, mode, nullptr, nullptr, ms);
}

int cs_match_mutual_host(void *h_s1, int n1, void *h_s2, int n2, float minScore, float maxAmbiguity, int *h_pairs,
                         int maxPairs, int mode, double *ms)
{
  if (ms) *ms = 0.0;
  int r = mutual_args("cs_match_mutual_host", h_s1, n1, h_s2, n2, h_pairs, maxPairs, mode);
  if (r < 0) return r;
  if (n1 == 0 || n2 == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const int room = maxPairs < (n1 < n2 ? n1 : n2) ? maxPairs : (n1 < n2 ? n1 : n2);   // no more pairs can exist
  return host_pairs(c, h_s1, n1, h_s2, n2, room > 0 ? room : 1, 0, room, h_pairs,
                    [&](SiftPoint *d1, SiftPoint *d2, int2 *pairs) {
                      const MutualArgs mu = {minScore, maxAmbiguity, pairs, room};
                      return match_sync("cs_match_mutual", d1, n1, d2, n2, &mu, mode, (SiftPoint *)h_s1,
                                        (SiftPoint *)h_s2, ms);
                    });
}

int cs_match_knn2(const void *d_s1, int n1, const void *d_s2, int n2, int *d_idx, float *d_score, int mode, double *ms)
{
  const char *fn = "cs_match_knn2";
  if (ms) *ms = 0.0;
  int r = check_sets(fn, d_s1, n1, d_s2, n2, mode);
  if (r < 0) return r;
  if ((r = knn_out_args(fn, d_s1, n1, d_s2, n2, d_idx, d_score)) < 0) return r;
  if (n1 == 0 || n2 == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  return knn_sync(fn, c, (const SiftPoint *)d_s1, n1, (const SiftPoint *)d_s2, n2, d_idx, d_score, nullptr, nullptr,
                  nullptr, mode, ms);
}

int cs_match_ratio(const void *d_s1, int n1, const void *d_s2, int n2, float maxRatio, float maxDistance, int crossCheck,
                   int *d_pairs, int maxPairs, int mode, double *ms)
{
  if (ms) *ms = 0.0;
  int r = ratio_args("cs_match_ratio", d_s1, n1, d_s2, n2, maxRatio, maxDistance, d_pairs, maxPairs, mode);
  if (r < 0) return r;
  if (n1 == 0 || n2 == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const RatioArgs ra = {maxRatio, maxDistance, (int2 *)d_pairs, maxPairs};
  return ratio_sync("cs_match_ratio", c, (const SiftPoint *)d_s1, n1, (const SiftPoint *)d_s2, n2, ra, crossCheck != 0,
                    mode, ms);
}

int cs_match_ratio_host(const void *h_s1, int n1, const void *h_s2, int n2, float maxRatio, float maxDistance,
                        int crossCheck, int *h_pairs, int maxPairs, int mode, double *ms)
{
  const char *fn = "cs_match_ratio_host";
  if (ms) *ms = 0.0;
  int r = ratio_args(fn, h_s1, n1, h_s2, n2, maxRatio, maxDistance, h_pairs, maxPairs, mode);
  if (r < 0) return r;
  if (n1 == 0 || n2 == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const int room = maxPairs < n1 ? maxPairs : n1;                      // at most one pair per row of set 1
  return host_pairs(c, h_s1, n1, h_s2, n2, room > 0 ? room : 1, 0, room, h_pairs,
                    [&](SiftPoint *d1, SiftPoint *d2, int2 *pairs) {
                      const RatioArgs ra = {maxRatio, maxDistance, pairs, room};
                      return ratio_sync(fn, c, d1, n1, d2, n2, ra, crossCheck != 0, mode, ms);
                    });
}

int cs_match_knn2_guided(const void *d_s1, int n1, const void *d_s2, int n2, int model, const double model_in[9],
                         float thresh, int *d_idx, float *d_score, double *ms)
{
  const char *fn = "cs_match_knn2_guided";
  if (ms) *ms = 0.0;
  int r = check_sets(fn, d_s1, n1, d_s2, n2, 0);                            // mode 0: one path
  if (r < 0) return r;
  if ((r = guided_args(fn, model, model_in, thresh)) < 0) return r;
  if ((r = knn_out_args(fn, d_s1, n1, d_s2, n2, d_idx, d_score)) < 0) return r;
  if (n1 == 0 || n2 == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  return guided_sync(fn, c, d_s1, n1, d_s2, n2, model, model_in, thresh, nullptr, false, d_idx, d_score, ms);
}

int cs_match_guided(const void *d_s1, int n1, const void *d_s2, int n2, int model, const double model_in[9],
                    float thresh, float maxRatio, float maxDistance, int crossCheck, int *d_pairs, int maxPairs,
                    double *ms)
{
  const char *fn = "cs_match_guided";
  if (ms) *ms = 0.0;
  int r = ratio_args(fn, d_s1, n1, d_s2, n2, maxRatio, maxDistance, d_pairs, maxPairs, 0);
  if (r < 0) return r;
  if ((r = guided_args(fn, model, model_in, thresh)) < 0) return r;
  if (n1 == 0 || n2 == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const RatioArgs ra = {maxRatio, maxDistance, (int2 *)d_pairs, maxPairs};
  return guided_sync(fn, c, d_s1, n1, d_s2, n2, model, model_in, thresh, &ra, crossCheck != 0, nullptr, nullptr, ms);
}

int cs_match_guided_host(const void *h_s1, int n1, const void *h_s2, int n2, int model, const double model_in[9],
                         float thresh, float maxRatio, float maxDistance, int crossCheck, int *h_pairs, int maxPairs,
                         double *ms)
{
  const char *fn = "cs_match_guided_host";
  if (ms) *ms = 0.0;
  int r = ratio_args(fn, h_s1, n1, h_s2, n2, maxRatio, maxDistance, h_pairs, maxPairs, 0);
  if (r < 0) return r;
  if ((r = guided_args(fn, model, model_in, thresh)) < 0) return r;
  if (n1 == 0 || n2 == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const int room = maxPairs < n1 ? maxPairs : n1;                      // at most one pair per row of set 1
  return host_pairs(c, h_s1, n1, h_s2, n2, room > 0 ? room : 1, 0, room, h_pairs,
                    [&](SiftPoint *d1, SiftPoint *d2, int2 *pairs) {
                      const RatioArgs ra = {maxRatio, maxDistance, pairs, room};
                      return guided_sync(fn, c, d1, n1, d2, n2, model, model_in, thresh, &ra, crossCheck != 0,
                                         nullptr, nullptr, ms);
                    });
}

int cs_match_guided_stats(unsigned long long out[4])
{
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  for (int i = 0; i < 4; i++) out[i] = c->guidedStats[i];
  return 0;
}

int cs_match_stats(unsigned long long out[4])
{
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  for (int i = 0; i < 4; i++) out[i] = c->matchStats[i];
  return 0;
}

int cs_verify_pairs(const void *d_s1, int n1, const void *d_s2, int n2, const int *d_pairs, int numPairs, int model,
                    int numLoops, float thresh, unsigned long long seed, double model_out[9], int *d_inliers,
                    int maxInliers, double *ms)
{
  const char *fn = "cs_verify_pairs";
  if (ms) *ms = 0.0;
  int r = verify_args(fn, d_s1, n1, d_s2, n2, d_pairs, numPairs, model, numLoops, thresh, model_out, d_inliers, maxInliers);
  if (r < 0) return r;
  for (int k = 0; k < 9; k++) model_out[k] = 0.0;
  if (numPairs == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const cs_verify_job job = verify_job((const SiftPoint *)d_s1, n1, (const SiftPoint *)d_s2, n2, d_pairs, numPairs, seed,
                                       d_inliers, maxInliers);
  if ((r = verify_batch_sync(fn, c, &job, 1, nullptr, model, numLoops, thresh, ms)) < 0) return r;
  return verify_result(*c, 0, numPairs, model_out, c->verifyStats);
}

int cs_verify_pairs_host(const void *h_s1, int n1, const void *h_s2, int n2, const int *h_pairs, int numPairs, int model,
                         int numLoops, float thresh, unsigned long long seed, double model_out[9], int *h_inliers,
                         int maxInliers, double *ms)
{
  const char *fn = "cs_verify_pairs_host";
  if (ms) *ms = 0.0;
  int r = verify_args(fn, h_s1, n1, h_s2, n2, h_pairs, numPairs, model, numLoops, thresh, model_out, h_inliers, maxInliers);
  if (r < 0) return r;
  for (int k = 0; k < 9; k++) model_out[k] = 0.0;
  if (numPairs == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  return verify_host_pairs(c, h_s1, n1, h_s2, n2, h_pairs, numPairs, seed, h_inliers, maxInliers,
                           [&](const cs_verify_job &job) {
                             const int q = verify_batch_sync(fn, c, &job, 1, nullptr, model, numLoops, thresh, ms);
                             return q < 0 ? q : verify_result(*c, 0, numPairs, model_out, c->verifyStats);
                           });
}

int cs_verify_stats(long long out[8])
{
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  for (int i = 0; i < 8; i++) out[i] = c->verifyStats[i];
  return 0;
}

int cs_verify_models(const void *d_s1, int n1, const void *d_s2, int n2, const int *d_pairs, int numPairs, int model,
                     int numLoops, float thresh, unsigned long long seed, double *h_models, int *h_counts,
                     double h_norm[5])
{
  const char *fn = "cs_verify_models";
  double dummy[9];
  int r = verify_args(fn, d_s1, n1, d_s2, n2, d_pairs, numPairs, model, numLoops, thresh, dummy, nullptr, 0);
  if (r < 0) return r;
  if (!h_models || !h_counts || !h_norm) return arg_error(fn, "NULL output array");
  if (numPairs == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const cs_verify_job job = verify_job((const SiftPoint *)d_s1, n1, (const SiftPoint *)d_s2, n2, d_pairs, numPairs, seed,
                                       nullptr, 0);
  return verify_models_sync(c, job, nullptr, model, numLoops, thresh, h_models, h_counts, h_norm);
}

static void essential_zero(double E[9], double R[9], double t[3])
{
  for (int k = 0; k < 9; k++) E[k] = R[k] = 0.0;
  for (int k = 0; k < 3; k++) t[k] = 0.0;
}

int cs_verify_essential(const void *d_s1, int n1, const void *d_s2, int n2, const int *d_pairs, int numPairs,
                        const double K1[9], const double K2[9], int numLoops, float thresh, unsigned long long seed,
                        double E_out[9], double R_out[9], double t_out[3], int *d_inliers, int maxInliers, double *ms)
{
  const char *fn = "cs_verify_essential";
  if (ms) *ms = 0.0;
  int r = essential_args(fn, d_s1, n1, d_s2, n2, d_pairs, numPairs, K1, K2, numLoops, thresh, E_out, R_out, t_out,
                         d_inliers, maxInliers);
  if (r < 0) return r;
  essential_zero(E_out, R_out, t_out);
  if (numPairs == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const VerifyCalib cal = verify_calib(K1, K2);
  const cs_verify_job job = verify_job((const SiftPoint *)d_s1, n1, (const SiftPoint *)d_s2, n2, d_pairs, numPairs, seed,
                                       d_inliers, maxInliers);
  if ((r = verify_batch_sync(fn, c, &job, 1, &cal, VERIFY_ESSENTIAL, numLoops, thresh, ms)) < 0) return r;
  return verify_essential_result(*c, 0, numPairs, E_out, R_out, t_out, c->essentialStats);
}

int cs_verify_essential_host(const void *h_s1, int n1, const void *h_s2, int n2, const int *h_pairs, int numPairs,
                             const double K1[9], const double K2[9], int numLoops, float thresh,
                             unsigned long long seed, double E_out[9], double R_out[9], double t_out[3],
                             int *h_inliers, int maxInliers, double *ms)
{
  const char *fn = "cs_verify_essential_host";
  if (ms) *ms = 0.0;
  int r = essential_args(fn, h_s1, n1, h_s2, n2, h_pairs, numPairs, K1, K2, numLoops, thresh, E_out, R_out, t_out,
                         h_inliers, maxInliers);
  if (r < 0) return r;
  essential_zero(E_out, R_out, t_out);
  if (numPairs == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const VerifyCalib cal = verify_calib(K1, K2);
  return verify_host_pairs(c, h_s1, n1, h_s2, n2, h_pairs, numPairs, seed, h_inliers, maxInliers,
                           [&](const cs_verify_job &job) {
                             const int q = verify_batch_sync(fn, c, &job, 1, &cal, VERIFY_ESSENTIAL, numLoops, thresh, ms);
                             return q < 0 ? q : verify_essential_result(*c, 0, numPairs, E_out, R_out, t_out,
                                                                        c->essentialStats);
                           });
}

int cs_verify_essential_stats(long long out[10])
{
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  for (int i = 0; i < 10; i++) out[i] = c->essentialStats[i];
  return 0;
}

int cs_verify_essential_models(const void *d_s1, int n1, const void *d_s2, int n2, const int *d_pairs, int numPairs,
                               const double K1[9], const double K2[9], int numLoops, float thresh,
                               unsigned long long seed, double *h_models, int *h_counts, double h_norm[5])
{
  const char *fn = "cs_verify_essential_models";
  double dummy[12];
  int r = essential_args(fn, d_s1, n1, d_s2, n2, d_pairs, numPairs, K1, K2, numLoops, thresh, dummy, dummy, dummy,
                         nullptr, 0);
  if (r < 0) return r;
  if (!h_models || !h_counts || !h_norm) return arg_error(fn, "NULL output array");
  if (numPairs == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const VerifyCalib cal = verify_calib(K1, K2);
  const cs_verify_job job = verify_job((const SiftPoint *)d_s1, n1, (const SiftPoint *)d_s2, n2, d_pairs, numPairs, seed,
                                       nullptr, 0);
  return verify_models_sync(c, job, &cal, VERIFY_ESSENTIAL, numLoops, thresh, h_models, h_counts, h_norm);
}

int cs_verify_pairs_batch(const cs_verify_job *jobs, int numJobs, int model, int numLoops, float thresh,
                          double *models_out, int *counts_out, long long *stats_out, double *ms)
{
  const char *fn = "cs_verify_pairs_batch";
  if (ms) *ms = 0.0;
  int r = verify_batch_args(fn, jobs, numJobs, model, numLoops, thresh, nullptr, nullptr, false);
  if (r < 0) return r;
  if (numJobs > 0 && (!models_out || !counts_out)) return arg_error(fn, "models_out and counts_out must not be NULL");
  return batch_body(fn, numJobs, counts_out, stats_out, 8, ms,
                    [&](int p) { for (int k = 0; k < 9; k++) models_out[9 * (size_t)p + k] = 0.0; },
                    [&](int p) { return jobs[p].numPairs > 0; },
                    [&](DeviceCtx *c) { return verify_enqueue(*c, jobs, numJobs, nullptr, model, numLoops, thresh, true); },
                    [&](DeviceCtx *c, int p, int q, long long *st) {
                      return verify_result(*c, q, jobs[p].numPairs, models_out + 9 * (size_t)p, st);
                    });
}

int cs_verify_essential_batch(const cs_verify_job *jobs, int numJobs, const double *K1s, const double *K2s,
                              int numLoops, float thresh, double *E_out, double *R_out, double *t_out,
                              int *counts_out, long long *stats_out, double *ms)
{
  const char *fn = "cs_verify_essential_batch";
  if (ms) *ms = 0.0;
  int r = verify_batch_args(fn, jobs, numJobs, CS_GEOM_FUNDAMENTAL, numLoops, thresh, K1s, K2s, true);
  if (r < 0) return r;
  if (numJobs > 0 && (!E_out || !R_out || !t_out || !counts_out))
    return arg_error(fn, "E_out, R_out, t_out and counts_out must not be NULL");
  std::vector<VerifyCalib> cal((size_t)numJobs);
  for (int p = 0; p < numJobs; p++) cal[p] = verify_calib(K1s + 9 * (size_t)p, K2s + 9 * (size_t)p);
  return batch_body(fn, numJobs, counts_out, stats_out, 10, ms,
                    [&](int p) { essential_zero(E_out + 9 * (size_t)p, R_out + 9 * (size_t)p, t_out + 3 * (size_t)p); },
                    [&](int p) { return jobs[p].numPairs > 0; },
                    [&](DeviceCtx *c) {
                      return verify_enqueue(*c, jobs, numJobs, cal.data(), VERIFY_ESSENTIAL, numLoops, thresh, true);
                    },
                    [&](DeviceCtx *c, int p, int q, long long *st) {
                      return verify_essential_result(*c, q, jobs[p].numPairs, E_out + 9 * (size_t)p,
                                                     R_out + 9 * (size_t)p, t_out + 3 * (size_t)p, st);
                    });
}

int cs_match_ratio_batch(const cs_match_set *sets, int numSets, const cs_match_job *jobs, int numJobs, float maxRatio,
                         float maxDistance, int crossCheck, int *counts_out, unsigned long long *stats_out, double *ms)
{
  const char *fn = "cs_match_ratio_batch";
  if (ms) *ms = 0.0;
  int r = ratio_batch_args(fn, sets, numSets, jobs, numJobs, maxRatio, maxDistance, counts_out);
  if (r < 0) return r;
  std::vector<RatioBatchOut> out((size_t)numJobs);
  return batch_body(fn, numJobs, counts_out, stats_out, 4, ms, [](int) {},
                    [&](int p) { return sets[jobs[p].set1].n > 0 && sets[jobs[p].set2].n > 0; },
                    [&](DeviceCtx *c) {
                      return ratio_batch_enqueue(*c, sets, numSets, jobs, numJobs, maxRatio, maxDistance, crossCheck != 0,
                                                 out.data());
                    },
                    [&](DeviceCtx *, int p, int, unsigned long long *st) {
                      const RatioBatchOut &o = out[p];
                      if (*o.bad1 || *o.bad2) {                             // as match_tensor_stats: all exact
                        st[0] = st[1] = 0; st[2] = ~0ull;
                      } else {
                        for (int k = 0; k < 2; k++) {
                          if (!o.counters[k]) continue;
                          st[0] += o.counters[k][1]; st[1] += o.counters[k][2]; st[2] += o.counters[k][0];
                        }
                      }
                      st[3] = 2;
                      return (int)*o.total;
                    });
}

int cs_match_guided_batch(const cs_match_set *sets, int numSets, const cs_match_job *jobs, int numJobs,
                          const int *models, const double *models_in, float thresh, float maxRatio, float maxDistance,
                          int crossCheck, int *counts_out, unsigned long long *stats_out, double *ms)
{
  const char *fn = "cs_match_guided_batch";
  if (ms) *ms = 0.0;
  int r = guided_batch_args(fn, sets, numSets, jobs, numJobs, models, models_in, thresh, maxRatio, maxDistance,
                            counts_out);
  if (r < 0) return r;
  std::vector<GuidedBatchOut> out((size_t)numJobs, GuidedBatchOut{nullptr, nullptr});
  return batch_body(fn, numJobs, counts_out, stats_out, 4, ms, [](int) {},
                    [&](int p) { return sets[jobs[p].set1].n > 0 && sets[jobs[p].set2].n > 0; },
                    [&](DeviceCtx *c) {
                      return guided_enqueue(*c, sets, jobs, numJobs, models, models_in, thresh, maxRatio, maxDistance,
                                            crossCheck != 0, out.data(), nullptr);
                    },
                    [&](DeviceCtx *, int p, int, unsigned long long *st) {
                      for (int k = 0; k < 4; k++) st[k] = out[p].stats[k];
                      return (int)*out[p].total;
                    });
}

int cs_build_tracks(const int *imageSizes, int numImages, const cs_track_list *lists, int numLists, int minLength,
                    int dropConflicting, int *d_trackOf, int *d_offsets, int maxTracks, int *d_members, int maxMembers,
                    long long stats_out[8], double *ms)
{
  const char *fn = "cs_build_tracks";
  if (ms) *ms = 0.0;
  int N = 0, P = 0;
  int r = tracks_args(fn, imageSizes, numImages, lists, numLists, minLength, d_trackOf, d_offsets, maxTracks, d_members,
                      maxMembers, &N, &P);
  if (r < 0) return r;
  if (stats_out)
    for (int k = 0; k < 8; k++) stats_out[k] = 0;
  const bool fillTrackOf = d_trackOf && N > 0;
  if (P == 0 && !fillTrackOf && !d_offsets) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if (P == 0) {                                                           // no pairs: no track, no launch
    if (fillTrackOf) CS_CUDA(cudaMemsetAsync(d_trackOf, 0xff, (size_t)N * sizeof(int), c->stream));
    if (d_offsets) CS_CUDA(cudaMemsetAsync(d_offsets, 0, sizeof(int), c->stream));
    CS_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
  }
  if ((r = timed_sync(fn, c, ms, [&] {
         return tracks_enqueue(*c, imageSizes, numImages, lists, numLists, minLength, dropConflicting != 0, d_trackOf,
                               d_offsets, maxTracks, d_members, maxMembers);
       })) < 0)
    return r;
  const unsigned long long *st = c->h_tracks.as<const unsigned long long>();
  if (stats_out)
    for (int k = 0; k < 8; k++) stats_out[k] = (long long)st[k];
  return (int)st[6];
}

int cs_vocab_assign(const cs_match_set *sets, int numSets, const void *d_vocab, int numWords, int *d_wordOf,
                    unsigned long long stats_out[5], double *ms)
{
  const char *fn = "cs_vocab_assign";
  if (ms) *ms = 0.0;
  int M = 0;
  int r = vocab_assign_args(fn, sets, numSets, d_vocab, numWords, d_wordOf, &M);
  if (r < 0) return r;
  if (stats_out)
    for (int k = 0; k < 5; k++) stats_out[k] = 0;
  if (M == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  VocabAssign va;
  if ((r = timed_sync(fn, c, ms, [&] {
         return vocab_assign_enqueue(*c, sets, numSets, d_vocab, numWords, d_wordOf, nullptr, va);
       })) < 0)
    return r;
  if (stats_out) vocab_assign_stats(va, stats_out);
  return 0;
}

int cs_vocab_train(const cs_match_set *sets, int numSets, int numWords, int maxIterations, unsigned long long seed,
                   void *d_vocab, double *trace_out, long long stats_out[4], double *ms)
{
  const char *fn = "cs_vocab_train";
  if (ms) *ms = 0.0;
  int M = 0;
  int r = vocab_train_args(fn, sets, numSets, numWords, maxIterations, d_vocab, &M);
  if (r < 0) return r;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  std::vector<double> trace((size_t)4 * maxIterations);
  long long st[4] = {0, 0, 0, 0};
  if ((r = timed_sync(fn, c, ms, [&] {
         return vocab_train(*c, sets, numSets, numWords, maxIterations, seed, static_cast<SiftPoint *>(d_vocab),
                            trace.data(), st);
       })) < 0)
    return r;
  if (trace_out) std::copy(trace.begin(), trace.end(), trace_out);
  if (stats_out)
    for (int k = 0; k < 4; k++) stats_out[k] = st[k];
  return (int)st[0];
}

int cs_retrieve_pairs(const int *imageSizes, int numImages, const int *d_wordOf, int numWords, int topK,
                      int *d_neighbours, double *d_scores, double *d_idf, int *d_pairs, int maxPairs,
                      long long stats_out[7], double *ms)
{
  const char *fn = "cs_retrieve_pairs";
  if (ms) *ms = 0.0;
  int N = 0;
  int r = retrieve_args(fn, imageSizes, numImages, d_wordOf, numWords, topK, d_neighbours, d_scores, d_idf, d_pairs,
                        maxPairs, &N);
  if (r < 0) return r;
  if (stats_out)
    for (int k = 0; k < 7; k++) stats_out[k] = 0;
  if (N == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if ((r = timed_sync(fn, c, ms, [&] {
         return retrieve_enqueue(*c, imageSizes, numImages, d_wordOf, numWords, topK, d_neighbours, d_scores, d_idf,
                                 d_pairs, maxPairs);
       })) < 0)
    return r;
  const unsigned long long *st = c->h_retrieve.as<const unsigned long long>();
  if (stats_out) {
    for (int k = 0; k < 7; k++) stats_out[k] = (long long)st[k];
    stats_out[4] = c->retrieveWaves;
  }
  return (int)st[5];
}

int cs_triangulate_tracks(const cs_match_set *sets, int numImages, const double *Ks, const double *Rs, const double *ts,
                          const int *d_offsets, int numTracks, const int *d_members, int numMembers, int numTrials,
                          double maxError, double minTriAngle, unsigned long long seed, double *d_points, int *d_counts,
                          float *d_errors, unsigned char *d_inlier, long long stats_out[8], double *ms)
{
  const char *fn = "cs_triangulate_tracks";
  if (ms) *ms = 0.0;
  int r = triangulate_args(fn, sets, numImages, Ks, Rs, ts, d_offsets, numTracks, d_members, numMembers, numTrials,
                           maxError, minTriAngle, d_points, d_counts, d_errors, d_inlier);
  if (r < 0) return r;
  if (stats_out)
    for (int k = 0; k < 8; k++) stats_out[k] = 0;
  if (numTracks == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if ((r = timed_sync(fn, c, ms, [&] {
         return triangulate_enqueue(*c, sets, numImages, Ks, Rs, ts, d_offsets, numTracks, d_members, numMembers,
                                    numTrials, maxError, minTriAngle, seed, d_points, d_counts, d_errors, d_inlier);
       })) < 0)
    return r;
  const unsigned long long *st = c->h_tri.as<const unsigned long long>();
  if (stats_out)
    for (int k = 0; k < 8; k++) stats_out[k] = (long long)st[k];
  return (int)st[5];
}

// K_out = Ks and dist_out = dists (zero for NULL dists), each when given.
static void bundle_intrinsics_unchanged(int numImages, const double *Ks, const double *dists, double *K_out,
                                        double *dist_out)
{
  if (K_out && K_out != Ks) memmove(K_out, Ks, (size_t)numImages * 9 * sizeof(double));
  if (dist_out && dist_out != dists) {
    if (dists) memmove(dist_out, dists, (size_t)numImages * 2 * sizeof(double));
    else memset(dist_out, 0, (size_t)numImages * 2 * sizeof(double));
  }
}

// cs_bundle_adjust and cs_bundle_adjust_intrinsics past their argument checks (fn names the call).
static int bundle_adjust_checked(const char *fn, const cs_match_set *sets, int numImages, const double *Ks,
                                 const double *dists, const unsigned char *refine, int loss, double lossScale,
                                 const double *Rs, const double *ts, const unsigned char *fixed, const int *d_offsets,
                                 int numTracks, const int *d_members, int numMembers, const unsigned char *d_use,
                                 double *d_points, int maxIterations, int maxLinearIterations, double linearTol,
                                 double maxError, double *K_out, double *dist_out, double *R_out, double *t_out,
                                 float *d_errors, unsigned char *d_inlier, double cost_out[2], double *trace_out,
                                 long long stats_out[8], double *ms)
{
  if (numTracks == 0) {
    bundle_intrinsics_unchanged(numImages, Ks, dists, K_out, dist_out);
    if (R_out != Rs) memmove(R_out, Rs, (size_t)numImages * 9 * sizeof(double));
    if (t_out != ts) memmove(t_out, ts, (size_t)numImages * 3 * sizeof(double));
    cost_out[0] = cost_out[1] = 0.0;
    if (trace_out)
      for (int k = 0; k < 4 * maxIterations; k++) trace_out[k] = 0.0;
    if (stats_out)
      for (int k = 0; k < 8; k++) stats_out[k] = 0;
    return 0;
  }
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  int r;
  if ((r = timed_sync(fn, c, ms, [&] {
         return bundle_enqueue(*c, sets, numImages, Ks, dists, refine, loss, lossScale, Rs, ts, fixed, d_offsets,
                               numTracks, d_members, numMembers, d_use, d_points, maxIterations, maxLinearIterations,
                               linearTol, maxError, d_errors, d_inlier);
       })) < 0)
    return r;
  // K and k come back from the device only when the call ran the 9-parameter block; else they are the input's
  const int nc = bundle_camera_block(numImages, dists, refine);
  if (nc == 6) bundle_intrinsics_unchanged(numImages, Ks, dists, K_out, dist_out);
  return bundle_result(*c, nc, numImages, maxIterations, K_out, dist_out, R_out, t_out, cost_out, trace_out,
                       stats_out);
}

int cs_bundle_adjust(const cs_match_set *sets, int numImages, const double *Ks, const double *Rs, const double *ts,
                     const unsigned char *fixed, const int *d_offsets, int numTracks, const int *d_members,
                     int numMembers, const unsigned char *d_use, double *d_points, int maxIterations,
                     int maxLinearIterations, double linearTol, double maxError, double *R_out, double *t_out,
                     float *d_errors, unsigned char *d_inlier, double cost_out[2], double *trace_out,
                     long long stats_out[8], double *ms)
{
  const char *fn = "cs_bundle_adjust";
  if (ms) *ms = 0.0;
  const int r = bundle_args(fn, sets, numImages, Ks, Rs, ts, fixed, d_offsets, numTracks, d_members, numMembers,
                            d_use, d_points, maxIterations, maxLinearIterations, linearTol, maxError, R_out, t_out,
                            d_errors, d_inlier, cost_out);
  if (r < 0) return r;
  return bundle_adjust_checked(fn, sets, numImages, Ks, nullptr, nullptr, 0, 1.0, Rs, ts, fixed, d_offsets, numTracks,
                               d_members, numMembers, d_use, d_points, maxIterations, maxLinearIterations, linearTol,
                               maxError, nullptr, nullptr, R_out, t_out, d_errors, d_inlier, cost_out, trace_out,
                               stats_out, ms);
}

int cs_bundle_adjust_intrinsics(const cs_match_set *sets, int numImages, const double *Ks, const double *dists,
                                const unsigned char *refine, int loss, double lossScale, const double *Rs,
                                const double *ts, const unsigned char *fixed, const int *d_offsets, int numTracks,
                                const int *d_members, int numMembers, const unsigned char *d_use, double *d_points,
                                int maxIterations, int maxLinearIterations, double linearTol, double maxError,
                                double *K_out, double *dist_out, double *R_out, double *t_out, float *d_errors,
                                unsigned char *d_inlier, double cost_out[2], double *trace_out, long long stats_out[8],
                                double *ms)
{
  const char *fn = "cs_bundle_adjust_intrinsics";
  if (ms) *ms = 0.0;
  int r = bundle_args(fn, sets, numImages, Ks, Rs, ts, fixed, d_offsets, numTracks, d_members, numMembers, d_use,
                      d_points, maxIterations, maxLinearIterations, linearTol, maxError, R_out, t_out, d_errors,
                      d_inlier, cost_out);
  if (r < 0) return r;
  r = bundle_intrinsics_args(fn, numImages, Ks, dists, refine, loss, lossScale, Rs, ts, K_out, dist_out, R_out, t_out);
  if (r < 0) return r;
  return bundle_adjust_checked(fn, sets, numImages, Ks, dists, refine, loss, lossScale, Rs, ts, fixed, d_offsets,
                               numTracks, d_members, numMembers, d_use, d_points, maxIterations, maxLinearIterations,
                               linearTol, maxError, K_out, dist_out, R_out, t_out, d_errors, d_inlier, cost_out,
                               trace_out, stats_out, ms);
}

int cs_undistort_records(const cs_match_set *sets, int numImages, const double *Ks, const double *dists,
                         void *const *d_out, double *ms)
{
  const char *fn = "cs_undistort_records";
  if (ms) *ms = 0.0;
  long long total = 0;
  int r = undistort_args(fn, sets, numImages, Ks, dists, d_out, &total);
  if (r < 0 || total == 0) return r;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if ((r = timed_sync(fn, c, ms, [&] { return undistort_enqueue(*c, sets, numImages, Ks, dists, d_out); })) < 0)
    return r;
  return 0;
}

int cs_rotation_averaging(int numImages, const int *edges, int numEdges, const double *Rrel, const double *weights,
                          int refImage, int maxIterations, int maxLinearIterations, double linearTol, double sigmaDeg,
                          double maxAngleDeg, double *R_out, double *residuals_out, unsigned char *inlier_out,
                          double cost_out[2], double *trace_out, long long stats_out[6], double ms_out[2])
{
  const char *fn = "cs_rotation_averaging";
  if (ms_out) ms_out[0] = ms_out[1] = 0.0;
  int r = rotavg_args(fn, numImages, edges, numEdges, Rrel, weights, refImage, maxIterations, maxLinearIterations,
                      linearTol, sigmaDeg, maxAngleDeg, R_out, residuals_out, inlier_out, cost_out, trace_out);
  if (r < 0) return r;
  if (numEdges == 0) {
    for (int a = 0; a < numImages; a++)
      for (int k = 0; k < 9; k++) R_out[9 * (size_t)a + k] = a == refImage ? (k % 4 == 0 ? 1.0 : 0.0) : NAN;
    cost_out[0] = cost_out[1] = 0.0;
    if (trace_out)
      for (int k = 0; k < 3 * maxIterations; k++) trace_out[k] = 0.0;
    if (stats_out)
      for (int k = 0; k < 6; k++) stats_out[k] = k == 2 ? 1 : 0;
    return 0;
  }
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const auto t0 = std::chrono::steady_clock::now();
  if ((r = rotavg_prepare(*c, numImages, edges, numEdges, Rrel, weights, refImage, maxIterations)) < 0) return r;
  if (ms_out) ms_out[0] = ms_since(t0);
  if ((r = timed_sync(fn, c, ms_out ? ms_out + 1 : nullptr, [&] {
         return rotavg_enqueue(*c, numImages, numEdges, maxIterations, maxLinearIterations, linearTol, sigmaDeg);
       })) < 0)
    return r;
  return rotavg_result(*c, numImages, numEdges, maxIterations, maxAngleDeg, R_out, residuals_out, inlier_out, cost_out,
                       trace_out, stats_out);
}

int cs_global_positioning(const cs_match_set *sets, int numImages, const double *Ks, const double *Rs,
                          const int *d_offsets, int numTracks, const int *d_members, int numMembers,
                          const unsigned char *d_use, int refImage, unsigned long long seed, int loss, double lossScale,
                          int maxIterations, int maxLinearIterations, double linearTol, double *t_out,
                          double *d_points, double cost_out[2], double *trace_out, long long stats_out[8], double *ms)
{
  const char *fn = "cs_global_positioning";
  if (ms) *ms = 0.0;
  int r = globalpos_args(fn, sets, numImages, Ks, Rs, d_offsets, numTracks, d_members, numMembers, d_use, refImage,
                         loss, lossScale, maxIterations, maxLinearIterations, linearTol, t_out, d_points, cost_out,
                         trace_out);
  if (r < 0) return r;
  if (numTracks == 0) {
    for (int k = 0; k < 3 * numImages; k++) t_out[k] = NAN;
    cost_out[0] = cost_out[1] = 0.0;
    if (trace_out)
      for (int k = 0; k < 4 * maxIterations; k++) trace_out[k] = 0.0;
    if (stats_out)
      for (int k = 0; k < 8; k++) stats_out[k] = 0;
    return 0;
  }
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if ((r = timed_sync(fn, c, ms, [&] {
         return globalpos_enqueue(*c, sets, numImages, Ks, Rs, d_offsets, numTracks, d_members, numMembers, d_use,
                                  refImage, seed, loss, lossScale, maxIterations, maxLinearIterations, linearTol,
                                  d_points);
       })) < 0)
    return r;
  return globalpos_result(*c, numImages, Rs, maxIterations, t_out, cost_out, trace_out, stats_out);
}

int cs_undistort_images(const cs_image *images, int numImages, const double *Ks, const double *dists,
                        float *const *d_out, long long *outside_out, double *ms)
{
  const char *fn = "cs_undistort_images";
  if (ms) *ms = 0.0;
  int r = undistort_images_args(fn, images, numImages, Ks, dists, d_out);
  if (r < 0 || numImages == 0) return r;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const unsigned long long *outside = nullptr;
  if ((r = timed_sync(fn, c, ms, [&] {
         return undistort_images_enqueue(*c, images, numImages, Ks, dists, d_out, &outside);
       })) < 0)
    return r;
  for (int a = 0; outside_out && a < numImages; a++) outside_out[a] = (long long)outside[a];
  return 0;
}

int cs_patch_match_stereo(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
                          const cs_stereo_job *jobs, int numJobs, int windowRadius, int windowStep, int numIterations,
                          int topK, unsigned long long seed, long long *stats_out, double *ms)
{
  const char *fn = "cs_patch_match_stereo";
  if (ms) *ms = 0.0;
  int r = patch_match_args(fn, images, numImages, Ks, Rs, ts, jobs, numJobs, windowRadius, windowStep, numIterations,
                           topK);
  if (r < 0 || numJobs == 0) return r;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const unsigned long long *counts = nullptr;
  if ((r = timed_sync(fn, c, ms, [&] {
         return patch_match_enqueue(*c, images, numImages, Ks, Rs, ts, jobs, numJobs, windowRadius, windowStep,
                                    numIterations, topK, seed, &counts);
       })) < 0)
    return r;
  for (int p = 0; stats_out && p < numJobs; p++) {
    const cs_image &I = images[jobs[p].ref];
    stats_out[3 * (size_t)p] = (long long)I.width * I.height;
    stats_out[3 * (size_t)p + 1] = (long long)counts[3 * (size_t)p + 1];
    stats_out[3 * (size_t)p + 2] = (long long)counts[3 * (size_t)p + 2];
  }
  return 0;
}

int cs_patch_match_stereo_geometric(const cs_image *images, int numImages, const double *Ks, const double *Rs,
                                    const double *ts, const cs_depth_prior *priors, const cs_stereo_job *jobs,
                                    int numJobs, int windowRadius, int windowStep, int numIterations, int topK,
                                    double geomWeight, double geomMaxError, unsigned long long seed,
                                    long long *stats_out, double *ms)
{
  const char *fn = "cs_patch_match_stereo_geometric";
  if (ms) *ms = 0.0;
  int r = patch_match_geometric_args(fn, images, numImages, Ks, Rs, ts, priors, jobs, numJobs, windowRadius,
                                     windowStep, numIterations, topK, geomWeight, geomMaxError);
  if (r < 0 || numJobs == 0) return r;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  const unsigned long long *counts = nullptr;
  if ((r = timed_sync(fn, c, ms, [&] {
         return patch_match_geometric_enqueue(*c, images, numImages, Ks, Rs, ts, priors, jobs, numJobs, windowRadius,
                                              windowStep, numIterations, topK, geomWeight, geomMaxError, seed,
                                              &counts);
       })) < 0)
    return r;
  const unsigned long long *extra = counts + 3 * (size_t)numJobs;
  for (int p = 0; stats_out && p < numJobs; p++) {
    const cs_image &I = images[jobs[p].ref];
    long long *st = stats_out + 5 * (size_t)p;
    st[0] = (long long)I.width * I.height;
    st[1] = (long long)counts[3 * (size_t)p + 1];
    st[2] = (long long)counts[3 * (size_t)p + 2];
    st[3] = (long long)extra[3 * (size_t)p];
    st[4] = (long long)extra[3 * (size_t)p + 1];
  }
  return 0;
}

int cs_fuse_depth_maps(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
                       const cs_stereo_job *jobs, int numJobs, float maxCost, int minConsistent, double maxReprojError,
                       double maxDepthError, double maxNormalErrorDeg, float *d_xyz, float *d_normal,
                       float *d_intensity, int *d_source, int maxPoints, long long stats_out[2], double *ms)
{
  const char *fn = "cs_fuse_depth_maps";
  if (ms) *ms = 0.0;
  if (stats_out) stats_out[0] = stats_out[1] = 0;
  int r = fuse_args(fn, images, numImages, Ks, Rs, ts, jobs, numJobs, maxCost, minConsistent, maxReprojError,
                    maxDepthError, maxNormalErrorDeg, d_xyz, d_normal, d_intensity, d_source, maxPoints);
  if (r < 0 || numJobs == 0) return r;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  unsigned int *total = nullptr;
  if ((r = timed_sync(fn, c, ms, [&] {
         return fuse_enqueue(*c, images, numImages, Ks, Rs, ts, jobs, numJobs, maxCost, minConsistent,
                             maxReprojError, maxDepthError, maxNormalErrorDeg, d_xyz, d_normal, d_intensity, d_source,
                             maxPoints, &total);
       })) < 0)
    return r;
  const int n = (int)*total;
  if (stats_out) {
    stats_out[0] = n;
    stats_out[1] = std::min(n, maxPoints);
  }
  return n;
}

int cs_poisson_mesh(const float *d_xyz, const float *d_normal, const float *d_intensity, int numPoints, int depth,
                    double scale, int maxIterations, double tol, double trim, float *d_vertices,
                    float *d_vertexIntensity, int maxVertices, int *d_triangles, int maxTriangles, float *d_chi,
                    double info_out[7], long long stats_out[10], double *ms)
{
  const char *fn = "cs_poisson_mesh";
  if (ms) *ms = 0.0;
  int r = mesh_args(fn, d_xyz, d_normal, d_intensity, numPoints, depth, scale, maxIterations, tol, trim, d_vertices,
                    d_vertexIntensity, maxVertices, d_triangles, maxTriangles, d_chi);
  if (r < 0) return r;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if ((r = c->h_mesh.grow(mesh_result_bytes())) < 0) return r;
  if ((r = timed_sync(fn, c, ms, [&] {
         return mesh_run(d_xyz, d_normal, d_intensity, numPoints, depth, scale, 0.0, maxIterations, tol, trim,
                         d_vertices, d_vertexIntensity, maxVertices, d_triangles, maxTriangles, d_chi, c->stream,
                         c->h_mesh.p);
       })) < 0)
    return r;
  return mesh_result(c->h_mesh.p, numPoints, maxVertices, maxTriangles, false, info_out, stats_out);
}

int cs_poisson_mesh_screened(const float *d_xyz, const float *d_normal, const float *d_intensity, int numPoints,
                             int depth, double scale, double pointWeight, int maxIterations, double tol, double trim,
                             float *d_vertices, float *d_vertexIntensity, int maxVertices, int *d_triangles,
                             int maxTriangles, float *d_chi, double info_out[8], long long stats_out[10], double *ms)
{
  const char *fn = "cs_poisson_mesh_screened";
  if (ms) *ms = 0.0;
  int r = mesh_screened_args(fn, d_xyz, d_normal, d_intensity, numPoints, depth, scale, pointWeight, maxIterations,
                             tol, trim, d_vertices, d_vertexIntensity, maxVertices, d_triangles, maxTriangles, d_chi);
  if (r < 0) return r;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if ((r = c->h_mesh.grow(mesh_result_bytes())) < 0) return r;
  if ((r = timed_sync(fn, c, ms, [&] {
         return mesh_run(d_xyz, d_normal, d_intensity, numPoints, depth, scale, pointWeight, maxIterations, tol, trim,
                         d_vertices, d_vertexIntensity, maxVertices, d_triangles, maxTriangles, d_chi, c->stream,
                         c->h_mesh.p);
       })) < 0)
    return r;
  return mesh_result(c->h_mesh.p, numPoints, maxVertices, maxTriangles, true, info_out, stats_out);
}

int cs_simplify_mesh(const float *d_vertices, const float *d_vertexIntensity, int numVertices, const int *d_triangles,
                     int numTriangles, int targetTriangles, double maxError, double boundaryWeight,
                     float *d_outVertices, float *d_outIntensity, int maxOutVertices, int *d_outTriangles,
                     int maxOutTriangles, double info_out[1], long long stats_out[9], double *ms)
{
  const char *fn = "cs_simplify_mesh";
  if (ms) *ms = 0.0;
  int r = simplify_args(fn, d_vertices, d_vertexIntensity, numVertices, d_triangles, numTriangles, targetTriangles,
                        maxError, boundaryWeight, d_outVertices, d_outIntensity, maxOutVertices, d_outTriangles,
                        maxOutTriangles);
  if (r < 0) return r;
  if (numTriangles == 0) {
    if (info_out) info_out[0] = 0.0;
    if (stats_out)
      for (int k = 0; k < 9; k++) stats_out[k] = 0;
    return 0;
  }
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if ((r = c->h_mesh.grow(simplify_result_bytes())) < 0) return r;
  return timed_sync(fn, c, ms, [&] {
    return simplify_run(d_vertices, d_vertexIntensity, numVertices, d_triangles, numTriangles, targetTriangles,
                        maxError, boundaryWeight, d_outVertices, d_outIntensity, maxOutVertices, d_outTriangles,
                        maxOutTriangles, c->stream, c->h_mesh.p, info_out, stats_out);
  });
}

int cs_clean_mesh(const float *d_vertices, const float *d_vertexIntensity, int numVertices, const int *d_triangles,
                  int numTriangles, int removeDegenerate, double longEdgeFactor, int removeNonManifold,
                  int minComponentFaces, double minComponentFraction, int maxHoleEdges, int smoothIterations,
                  double lambda, double mu, float *d_outVertices, float *d_outIntensity, int maxOutVertices,
                  int *d_outTriangles, int maxOutTriangles, double info_out[3], long long stats_out[19], double *ms)
{
  const char *fn = "cs_clean_mesh";
  if (ms) *ms = 0.0;
  int r = clean_args(fn, d_vertices, d_vertexIntensity, numVertices, d_triangles, numTriangles, removeDegenerate,
                     longEdgeFactor, removeNonManifold, minComponentFaces, minComponentFraction, maxHoleEdges,
                     smoothIterations, lambda, mu, d_outVertices, d_outIntensity, maxOutVertices, d_outTriangles,
                     maxOutTriangles);
  if (r < 0) return r;
  if (numTriangles == 0) {
    if (info_out)
      for (int k = 0; k < 3; k++) info_out[k] = 0.0;
    if (stats_out)
      for (int k = 0; k < 19; k++) stats_out[k] = 0;
    return 0;
  }
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if ((r = c->h_mesh.grow(clean_result_bytes())) < 0) return r;
  return timed_sync(fn, c, ms, [&] {
    return clean_run(d_vertices, d_vertexIntensity, numVertices, d_triangles, numTriangles, removeDegenerate,
                     longEdgeFactor, removeNonManifold, minComponentFaces, minComponentFraction, maxHoleEdges,
                     smoothIterations, lambda, mu, d_outVertices, d_outIntensity, maxOutVertices, d_outTriangles,
                     maxOutTriangles, c->stream, c->h_mesh.p, info_out, stats_out);
  });
}

int cs_texture_mesh(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
                    const float *d_vertices, int numVertices, const int *d_triangles, int numTriangles, double lambda,
                    double maxViewAngleDeg, double depthTol, int padding, int atlasWidth, int maxSweeps,
                    float *d_atlas, int maxAtlasRows, float *d_uv, int *d_faceView, int *d_faceChart,
                    int *charts_out, int maxCharts, double info_out[2], long long stats_out[11], double *ms)
{
  const char *fn = "cs_texture_mesh";
  if (ms) *ms = 0.0;
  int r = texture_args(fn, images, numImages, Ks, Rs, ts, d_vertices, numVertices, d_triangles, numTriangles, lambda,
                       maxViewAngleDeg, depthTol, padding, atlasWidth, maxSweeps, d_atlas, maxAtlasRows, d_uv,
                       d_faceView, d_faceChart, charts_out, maxCharts);
  if (r < 0) return r;
  if (numTriangles == 0) {
    if (info_out) info_out[0] = info_out[1] = 0.0;
    if (stats_out)
      for (int k = 0; k < 11; k++) stats_out[k] = 0;
    return 0;
  }
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if ((r = c->h_mesh.grow(texture_result_bytes())) < 0) return r;
  return timed_sync(fn, c, ms, [&] {
    return texture_run(images, numImages, Ks, Rs, ts, d_vertices, numVertices, d_triangles, numTriangles, lambda,
                       maxViewAngleDeg, depthTol, padding, atlasWidth, maxSweeps, d_atlas, maxAtlasRows, d_uv,
                       d_faceView, d_faceChart, charts_out, maxCharts, c->stream, c->h_mesh.p, info_out, stats_out);
  });
}

int cs_texture_mesh_photo(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
                          const float *d_vertices, int numVertices, const int *d_triangles, int numTriangles,
                          int dataTerm, double outlierK, double outlierMinSigma, double lambda,
                          double maxViewAngleDeg, double depthTol, int padding, int atlasWidth, int maxSweeps,
                          float *d_atlas, int maxAtlasRows, float *d_uv, int *d_faceView, int *d_faceChart,
                          int *charts_out, int maxCharts, double info_out[2], long long stats_out[16], double *ms)
{
  const char *fn = "cs_texture_mesh_photo";
  if (ms) *ms = 0.0;
  int r = texture_args(fn, images, numImages, Ks, Rs, ts, d_vertices, numVertices, d_triangles, numTriangles, lambda,
                       maxViewAngleDeg, depthTol, padding, atlasWidth, maxSweeps, d_atlas, maxAtlasRows, d_uv,
                       d_faceView, d_faceChart, charts_out, maxCharts);
  if (r < 0 || (r = texture_photo_args(fn, dataTerm, outlierK, outlierMinSigma)) < 0) return r;
  if (numTriangles == 0) {
    if (info_out) info_out[0] = info_out[1] = 0.0;
    if (stats_out)
      for (int k = 0; k < 16; k++) stats_out[k] = 0;
    return 0;
  }
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if ((r = c->h_mesh.grow(texture_result_bytes())) < 0) return r;
  const TexturePhoto photo{dataTerm, outlierK, outlierMinSigma};
  return timed_sync(fn, c, ms, [&] {
    return texture_run(images, numImages, Ks, Rs, ts, d_vertices, numVertices, d_triangles, numTriangles, lambda,
                       maxViewAngleDeg, depthTol, padding, atlasWidth, maxSweeps, d_atlas, maxAtlasRows, d_uv,
                       d_faceView, d_faceChart, charts_out, maxCharts, c->stream, c->h_mesh.p, info_out, stats_out,
                       &photo);
  });
}

int cs_texture_mesh_bp(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
                       const float *d_vertices, int numVertices, const int *d_triangles, int numTriangles,
                       int dataTerm, double outlierK, double outlierMinSigma, int maxBpSweeps, double lambda,
                       double maxViewAngleDeg, double depthTol, int padding, int atlasWidth, int maxSweeps,
                       float *d_atlas, int maxAtlasRows, float *d_uv, int *d_faceView, int *d_faceChart,
                       int *charts_out, int maxCharts, double info_out[3], long long stats_out[20], double *ms)
{
  const char *fn = "cs_texture_mesh_bp";
  if (ms) *ms = 0.0;
  int r = texture_args(fn, images, numImages, Ks, Rs, ts, d_vertices, numVertices, d_triangles, numTriangles, lambda,
                       maxViewAngleDeg, depthTol, padding, atlasWidth, maxSweeps, d_atlas, maxAtlasRows, d_uv,
                       d_faceView, d_faceChart, charts_out, maxCharts);
  if (r < 0 || (r = texture_photo_args(fn, dataTerm, outlierK, outlierMinSigma)) < 0 ||
      (r = texture_bp_args(fn, maxBpSweeps)) < 0)
    return r;
  if (numTriangles == 0) {
    if (info_out) info_out[0] = info_out[1] = info_out[2] = 0.0;
    if (stats_out)
      for (int k = 0; k < 20; k++) stats_out[k] = 0;
    return 0;
  }
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if ((r = c->h_mesh.grow(texture_result_bytes())) < 0) return r;
  const TexturePhoto photo{dataTerm, outlierK, outlierMinSigma};
  return timed_sync(fn, c, ms, [&] {
    return texture_run(images, numImages, Ks, Rs, ts, d_vertices, numVertices, d_triangles, numTriangles, lambda,
                       maxViewAngleDeg, depthTol, padding, atlasWidth, maxSweeps, d_atlas, maxAtlasRows, d_uv,
                       d_faceView, d_faceChart, charts_out, maxCharts, c->stream, c->h_mesh.p, info_out, stats_out,
                       &photo, maxBpSweeps);
  });
}

int cs_mesh_refine(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
                   const float *d_vertices, int numVertices, const int *d_triangles, int numTriangles,
                   const int *pairs, int numPairs, int windowRadius, double smoothness, double step,
                   int maxIterations, double depthTol, float *d_outVertices, double info_out[4],
                   long long stats_out[8], double *ms)
{
  const char *fn = "cs_mesh_refine";
  if (ms) *ms = 0.0;
  int r = refine_args(fn, images, numImages, Ks, Rs, ts, d_vertices, numVertices, d_triangles, numTriangles, pairs,
                      numPairs, windowRadius, smoothness, step, maxIterations, depthTol, d_outVertices);
  if (r < 0) return r;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if (numTriangles == 0) {
    // no face: every vertex is fixed and copied, status 1
    if (info_out)
      for (int k = 0; k < 4; k++) info_out[k] = 0.0;
    if (stats_out) {
      const long long s[8] = {numPairs, 0, numVertices, 0, 0, 0, 0, 1};
      for (int k = 0; k < 8; k++) stats_out[k] = s[k];
    }
    return timed_sync(fn, c, ms, [&]() -> int {
      if (numVertices)
        CS_CUDA(cudaMemcpyAsync(d_outVertices, d_vertices, (size_t)numVertices * 12, cudaMemcpyDeviceToDevice,
                                c->stream));
      return 1;
    });
  }
  if ((r = c->h_mesh.grow(refine_result_bytes())) < 0) return r;
  return timed_sync(fn, c, ms, [&] {
    return refine_run(images, numImages, Ks, Rs, ts, d_vertices, numVertices, d_triangles, numTriangles, pairs,
                      numPairs, windowRadius, smoothness, step, maxIterations, depthTol, d_outVertices, c->stream,
                      c->h_mesh.p, info_out, stats_out);
  });
}

int cs_level_texture_seams(const float *d_vertices, int numVertices, const int *d_triangles, int numTriangles,
                           const int *d_faceView, const float *d_uv, const int *charts, int numCharts,
                           const float *d_atlas, int atlasRows, int atlasWidth, int padding, double smoothness,
                           double regularization, int maxIterations, double tol, float *d_outAtlas,
                           float *d_cornerOffset, double info_out[3], long long stats_out[8], double *ms)
{
  const char *fn = "cs_level_texture_seams";
  if (ms) *ms = 0.0;
  int r = seams_args(fn, d_vertices, numVertices, d_triangles, numTriangles, d_faceView, d_uv, charts, numCharts,
                     d_atlas, atlasRows, atlasWidth, padding, smoothness, regularization, false, 0, maxIterations,
                     tol, d_outAtlas, d_cornerOffset);
  if (r < 0) return r;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if ((r = c->h_mesh.grow(seams_result_bytes())) < 0) return r;
  return timed_sync(fn, c, ms, [&] {
    return seams_run(d_vertices, numVertices, d_triangles, numTriangles, d_faceView, d_uv, charts, numCharts, d_atlas,
                     atlasRows, atlasWidth, padding, smoothness, regularization, maxIterations, tol, d_outAtlas,
                     d_cornerOffset, c->stream, c->h_mesh.p, info_out, stats_out);
  });
}

int cs_level_texture_seams_local(const float *d_vertices, int numVertices, const int *d_triangles, int numTriangles,
                                 const int *d_faceView, const float *d_uv, const int *charts, int numCharts,
                                 const float *d_atlas, int atlasRows, int atlasWidth, int padding, int stripWidth,
                                 int maxIterations, double tol, float *d_outAtlas, double info_out[3],
                                 long long stats_out[8], double *ms)
{
  const char *fn = "cs_level_texture_seams_local";
  if (ms) *ms = 0.0;
  int r = seams_args(fn, d_vertices, numVertices, d_triangles, numTriangles, d_faceView, d_uv, charts, numCharts,
                     d_atlas, atlasRows, atlasWidth, padding, 0.0, 0.0, true, stripWidth, maxIterations, tol,
                     d_outAtlas, nullptr);
  if (r < 0) return r;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if ((r = c->h_mesh.grow(seams_local_result_bytes())) < 0) return r;
  return timed_sync(fn, c, ms, [&] {
    return seams_local_run(d_vertices, numVertices, d_triangles, numTriangles, d_faceView, d_uv, charts, numCharts,
                           d_atlas, atlasRows, atlasWidth, padding, stripWidth, maxIterations, tol, d_outAtlas,
                           c->stream, c->h_mesh.p, info_out, stats_out);
  });
}

int cs_absolute_pose_batch(const double *d_points, int numPoints, const cs_pose_job *jobs, int numJobs,
                           const double *Ks, int numLoops, double maxError, double *R_out, double *t_out,
                           int *counts_out, long long *stats_out, double *ms)
{
  const char *fn = "cs_absolute_pose_batch";
  if (ms) *ms = 0.0;
  int r = pose_args(fn, d_points, numPoints, jobs, numJobs, Ks, numLoops, maxError);
  if (r < 0) return r;
  if (numJobs > 0 && (!R_out || !t_out || !counts_out)) return arg_error(fn, "R_out, t_out and counts_out must not be NULL");
  r = batch_body(fn, numJobs, counts_out, stats_out, 8, ms,
                 [&](int p) {
                   for (int k = 0; k < 9; k++) R_out[9 * (size_t)p + k] = 0.0;
                   for (int k = 0; k < 3; k++) t_out[3 * (size_t)p + k] = 0.0;
                 },
                 [&](int p) { return jobs[p].n > 0; },
                 [&](DeviceCtx *c) { return pose_enqueue(*c, d_points, numPoints, jobs, numJobs, Ks, numLoops, maxError, true); },
                 [&](DeviceCtx *c, int p, int q, long long *st) {
                   return pose_result(*c, q, R_out + 9 * (size_t)p, t_out + 3 * (size_t)p, st);
                 });
  if (r < 0) return r;
  int posed = 0;
  for (int p = 0; p < numJobs; p++) posed += counts_out[p] > 0;
  return posed;
}

int cs_absolute_pose_models(const double *d_points, int numPoints, const cs_pose_job *job, const double K[9],
                            int numLoops, double maxError, double *h_R, double *h_t, int *h_counts)
{
  const char *fn = "cs_absolute_pose_models";
  int r = pose_args(fn, d_points, numPoints, job, job ? 1 : 0, K, numLoops, maxError);
  if (r < 0) return r;
  if (!job) return arg_error(fn, "job must not be NULL");
  if (!h_R || !h_t || !h_counts) return arg_error(fn, "NULL output array");
  if (job->n == 0) return 0;
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if ((r = pose_enqueue(*c, d_points, numPoints, job, 1, K, numLoops, maxError, false)) < 0) return r;
  return pose_models_to_host(*c, *job, numLoops, h_R, h_t, h_counts);
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

int cs_describe_points(const float *d_img, int w, int h, int pitch, void *d_pts, int n, int maxPts,
                       float finestSubsampling)
{
  if (!d_img || !d_pts || w < 1 || h < 1 || pitch < w || maxPts < 1 || n < 0 || n > maxPts) {
    set_error("cs_describe_points: invalid argument (CS_E_ARG)");
    return CS_E_ARG;
  }
  int err = 0;
  DeviceCtx *c = current_ctx(&err);
  if (!c) return err;
  if (n == 0) return 0;
  // describe_kernel picks the texture by log2(subsampling): refuse records it cannot index
  std::vector<float> sub(n);
  CS_CUDA(cudaMemcpy2D(sub.data(), sizeof(float), (const char *)d_pts + offsetof(SiftPoint, subsampling),
                       sizeof(SiftPoint), sizeof(float), n, cudaMemcpyDeviceToHost));
  for (int i = 0; i < n; i++) {
    int e = 0;
    if (!(std::frexp(sub[i], &e) == 0.5f && e >= 1 && e <= CS_MAX_LEVELS)) {
      set_error("cs_describe_points: record %d has subsampling %g, not 2^k with 0 <= k < %d", i, sub[i], CS_MAX_LEVELS);
      return CS_E_ARG;
    }
  }
  DescribeParams ds;
  memset(&ds, 0, sizeof(ds));
  cudaTextureObject_t tex = 0;
  int r = make_texture(&tex, d_img, w, h, pitch);
  if (r < 0) return r;
  for (int i = 0; i < CS_MAX_LEVELS; i++) ds.tex[i] = tex;
  unsigned int *d_cnt = nullptr;
  const unsigned int cnt0[CS_CNT_STRIDE + 1] = {(unsigned)n, 0u, 0u, 0u, 0u};   // counters | queue word
  cudaError_t e = cudaMalloc((void **)&d_cnt, sizeof(cnt0));
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_cnt, cnt0, sizeof(cnt0), cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess) {
    ds.numLevels = CS_MAX_LEVELS; ds.numImages = 1; ds.pts = (SiftPoint *)d_pts; ds.counters = d_cnt; ds.maxPts = maxPts;
    ds.finestSubsampling = finestSubsampling;
    ds.queue = d_cnt + CS_CNT_STRIDE;
    r = launch_describe(ds, c->stream);
    if (r == 0) e = cudaMemcpyAsync(c->h_counters, d_cnt, 2 * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream);
    if (r == 0 && e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
  }
  if (d_cnt) cudaFree(d_cnt);
  cudaDestroyTextureObject(tex);
  if (r < 0) return r;
  CS_CUDA(e);
  return count_from_counters(c->h_counters, maxPts);
}

// ---- pipelined extractor ----
struct cs_extractor {
  int w = 0, h = 0, numOctaves = 0, maxPts = 0, scaleUp = 0, pitch = 0, B = 0;
  cudaStream_t stream = nullptr;
  bool legacy = false;             // the round-1 per-image kernels (B == 1)
  Pipeline pipe;
  float *d_img = nullptr;          // B staging images
  SiftPoint *d_pts = nullptr;      // B x maxPts records (ranked: the output slots)
  int maxCand = 0;                 // ranked extractors: candidate records per image (0: plain extractor)
  SiftPoint *d_cand = nullptr;     // ranked: B x maxCand records, written by the pipeline as d_pts is for a plain extractor
  unsigned int *d_rank = nullptr;  // ranked: B x rank_scratch_words(maxCand)
  float *h_img = nullptr;          // pinned, B x w x h
  uint8_t *d_u8 = nullptr;         // device staging for 8-bit uploads (lazily allocated)
  SiftPoint *h_pts = nullptr;      // pinned, B x maxPts
  unsigned int *h_counters = nullptr;   // pinned, B x CS_CNT_STRIDE
  bool hostResults = false;
  int lastN = 0;
  int lastCounts[CS_MAX_BATCH] = {};
  int lastCand[CS_MAX_BATCH] = {};      // records found per image (ranked: in the candidate area)
  // CUDA graph of one steady-state submit of the batched kernels (memset + kernels + count D2H).  Per submit only the
  // input images change: the tensor maps in the parameters of the first pyramid kernel, patched with
  // cudaGraphExecKernelNodeSetParams.
  cudaGraphExec_t gexec = nullptr;
  cudaGraph_t graph = nullptr;
  cudaGraphNode_t gnode = nullptr;
  cudaKernelNodeParams gparams = {};
  PyrAParams gpa = {};
  int gn = 0, gpitch = 0, glaunches = 0;
  double gblur = 0.0;
  float gthresh = 0.0f, glowest = 0.0f;
  int submits = 0;
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
    r = ex->pipe.enqueue_round1(d_imgs[0], pitch, initBlur, thresh, lowestScale, ex->d_pts, ex->maxPts, ex->stream, ev);
  } else if (ex->maxCand > 0) {
    RankParams rp;
    memset(&rp, 0, sizeof(rp));
    rp.out = ex->d_pts; rp.outStride = ex->maxPts; rp.maxOut = ex->maxPts; rp.scratch = ex->d_rank;
    r = ex->pipe.enqueue(n, d_imgs, pitch, initBlur, thresh, lowestScale, ex->d_cand, ex->maxCand, ex->maxCand, ex->stream,
                         ev, paOut, &rp);
  } else {
    r = ex->pipe.enqueue(n, d_imgs, pitch, initBlur, thresh, lowestScale, ex->d_pts, ex->maxPts, ex->maxPts, ex->stream, ev, paOut);
  }
  if (r < 0) return r;
  CS_CUDA(cudaMemcpyAsync(ex->h_counters, ex->pipe.counters(0), (size_t)n * CS_CNT_STRIDE * sizeof(unsigned int),
                          cudaMemcpyDeviceToHost, ex->stream));
  return 0;
}

// Capture one submit of the batched kernels into a graph.  Leaves ex->gexec == NULL if anything is unsupported (the
// up-scaled and the round-1 pipelines are not captured); the caller then launches directly.
static int extractor_capture(cs_extractor *ex, int n, const float *const *d_imgs, int pitch, double initBlur, float thresh,
                             float lowestScale)
{
  if (ex->scaleUp || ex->legacy) return 0;
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
    if (kp.func == cs::pyr_a_func()) {
      ex->gnode = nodes[i]; ex->gparams = kp;
      found = true;
    }
  }
  cudaGraphExec_t ge = nullptr;
  if (!found || cudaGraphInstantiate(&ge, g, 0) != cudaSuccess) { cudaGetLastError(); cudaGraphDestroy(g); return 0; }
  ex->graph = g; ex->gexec = ge;
  ex->gn = n; ex->gpitch = pitch; ex->gblur = initBlur; ex->gthresh = thresh; ex->glowest = lowestScale;
  return 0;
}

static cs_extractor *extractor_create(int w, int h, int numOctaves, int maxPts, int scaleUp, int batch, int maxCand)
{
  if (batch < 1 || batch > CS_MAX_BATCH) { set_error("cs_extractor_create_batch: batch %d out of range (1..%d)", batch, CS_MAX_BATCH); return nullptr; }
  if (check_level0_size("cs_extractor_create", w, h, scaleUp != 0) < 0) return nullptr;
  cs_extractor *ex = new cs_extractor();
  ex->w = w; ex->h = h; ex->numOctaves = numOctaves; ex->maxPts = maxPts; ex->scaleUp = scaleUp; ex->B = batch;
  ex->pitch = ialignup(w, 128);
  ex->legacy = legacy_mode();
  if (ex->legacy && batch != 1) { set_error("the legacy pipeline takes one image at a time"); delete ex; return nullptr; }
  bool ok = cudaStreamCreateWithFlags(&ex->stream, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && ex->pipe.init(w, h, numOctaves, scaleUp != 0, batch, nullptr) == 0;
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
    int r = ex->pipe.fill_pyr_a(ex->gpa, n, d_imgs, pitch, initBlur);
    if (r < 0) return r;
    cudaKernelNodeParams kp = ex->gparams;
    void *args[1] = {(void *)&ex->gpa};
    kp.kernelParams = args;
    CS_CUDA(cudaGraphExecKernelNodeSetParams(ex->gexec, ex->gnode, &kp));
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
  if (slot < 0 || slot >= ex->B || level < 0 || level >= ex->pipe.numLevels) { set_error("cs_extractor_read_level: bad level"); return CS_E_ARG; }
  const float *src = ex->pipe.level(slot, level);
  const int lw = ex->pipe.lw[level], lh = ex->pipe.lh[level], lp = ex->pipe.lp[level];
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
  const size_t words = CS_CNT_STRIDE + rank_scratch_words(n);   // counters | scratch
  int r = c->rank.grow(words * sizeof(unsigned int));
  if (r < 0) return r;
  unsigned int *cnt = c->rank.as<unsigned int>();
  const unsigned int init[CS_CNT_STRIDE] = {(unsigned)n, (unsigned)n, 0u, 0u};
  CS_CUDA(cudaMemcpyAsync(cnt, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
  RankParams rp;
  memset(&rp, 0, sizeof(rp));
  rp.in = (const SiftPoint *)d_in; rp.maxIn = n;
  rp.out = (SiftPoint *)d_out; rp.maxOut = maxOut;
  rp.counters = cnt; rp.scratch = cnt + CS_CNT_STRIDE;
  if ((r = launch_rank(rp, 1, c->sms, c->stream)) < 0) return r;
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
