// common.cuh -- internal declarations shared by the cudasift_b200 translation units.
#pragma once

#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <algorithm>
#include <functional>
#include <map>
#include <vector>

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

// One resident wave of Kernel at Threads per CTA and no dynamic shared memory: the CTAs an SM holds at once (at least
// one) times the SM count, queried once per device; CS_E_CUDA when a query fails.
template <auto Kernel, int Threads>
int resident_grid()
{
  static int gridOf[64];
  int dev = 0;
  CS_CUDA(cudaGetDevice(&dev));
  dev &= 63;
  if (gridOf[dev] == 0) {
    int sms = 0, perSm = 0;
    CS_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    CS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, Kernel, Threads, 0));
    gridOf[dev] = (perSm > 0 ? perSm : 1) * sms;
  }
  return gridOf[dev];
}

// resident_grid for a cooperative kernel, after the check that the device supports cooperative launches: CS_E_CUDA,
// with call's name in the message, when it does not.
template <auto Kernel, int Threads>
int coop_grid(const char *call)
{
  int dev = 0, coop = 0;
  CS_CUDA(cudaGetDevice(&dev));
  CS_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  if (!coop) {
    set_error("%s: device %d does not support cooperative launches", call, dev);
    return CS_E_CUDA;
  }
  return resident_grid<Kernel, Threads>();
}

// The key bits of a radix sort whose keys are at most maxKey: the smallest bits (1 to 31) with maxKey < 2^bits.
inline int radix_bits(long long maxKey)
{
  int bits = 1;
  while (bits < 31 && (1ll << bits) <= maxKey) bits++;
  return bits;
}

// The ordered key of a float: keys compare as unsigned integers in the order of the floats they encode (finite values;
// -0 before +0), so an integer atomicMax of keys is a max of the floats (mesh.cu's box, match_guided.cu's index box).
__device__ __forceinline__ unsigned int float_key(float f)
{
  const unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(unsigned int k)
{
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

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
// Widest and tallest level 0 (after scaleUp) the detector takes: an extremum's tag (detect2.cu, cap32.cu) packs gx and gy
// into 13 bits each, and interior pixels reach w - 2 and h - 2.
#define CS_MAX_LEVEL0 8193

// ---- orientation + descriptor ---------------------------------------------------------
struct DescribeParams {
  cudaTextureObject_t tex[CS_MAX_LEVELS];   // indexed by log2(subsampling); used when texArr == NULL
  const cudaTextureObject_t *texArr;        // batch: [image * CS_MAX_LEVELS + level] (device memory)
  int numLevels;
  int numImages;                            // 1..CS_MAX_BATCH
  SiftPoint *pts;                           // image i: pts + i * ptsStride
  long long ptsStride;
  unsigned int *counters;                   // image i: counters + i * cntStride
  int cntStride;
  int maxPts;
  float finestSubsampling;  // secondaries of this level are dropped (reference quirk Q1)
  unsigned int *queue;      // keypoint queue counter of all images (zero before the launch)
};
int launch_describe(const DescribeParams &p, cudaStream_t st);
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

// ---- per-device context ---------------------------------------------------------------------------------------------
// A device buffer that grows on demand: grow() keeps the allocation when it holds `bytes`, else replaces it (the
// contents are not kept).
struct GrowBuffer {
  void *p = nullptr;
  size_t cap = 0;
  int grow(size_t bytes)
  {
    if (cap >= bytes) return 0;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    CS_CUDA(cudaMalloc(&p, bytes));
    cap = bytes;
    return 0;
  }
  template <class T> T *as() const { return static_cast<T *>(p); }
};
// The same in pinned host memory.  Every call that copies into or out of one ends in a synchronize, so no copy is
// pending when the next call grows it.
struct PinnedBuffer {
  void *p = nullptr;
  size_t cap = 0;
  int grow(size_t bytes)
  {
    if (cap >= bytes) return 0;
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    CS_CUDA(cudaMallocHost(&p, bytes));
    cap = bytes;
    return 0;
  }
  template <class T> T *as() const { return static_cast<T *>(p); }
};

// Consecutive pieces of one allocation: take(n) returns the next piece's offset and moves on by n rounded up to align
// (a power of two); bytes is the size of the pieces taken so far.
struct Layout {
  size_t align, bytes = 0;
  explicit Layout(size_t a) : align(a) {}
  size_t take(size_t n)
  {
    const size_t at = bytes;
    bytes += (n + align - 1) & ~(align - 1);
    return at;
  }
};

// The scratch budget of one wave of a batched call: RANSAC model slots (verify.cu, pose.cu), ratio and guided matching
// (match_tc.cu, match_guided.cu) and retrieval query accumulators (vocab.cu).  The header states each call's rule.
constexpr size_t WAVE_BYTES = (size_t)256 << 20;

// ---- the waves of a batched RANSAC call (verify.cu, pose.cu) --------------------------------------------------------
// A wave holds floor(WAVE_BYTES / slotBytes) jobs, slotBytes being one job's model slots and their counts, clamped to
// [1, 65536].
inline int ransac_jobs_per_wave(size_t slotBytes)
{
  const size_t k = WAVE_BYTES / slotBytes;
  return k < 1 ? 1 : k > 65536 ? 65536 : (int)k;
}

// The waves of a batch: its non-empty jobs (extent > 0) in input order (live[q] is the input index of the q-th), cut
// into runs of perWave jobs (the last run may be shorter); extent is the largest sum of the per-job extents of a wave.
struct WavePlan {
  std::vector<int> live;
  int perWave = 1;
  size_t extent = 0;
};
template <class Job, class Extent>
WavePlan wave_plan(const Job *jobs, int numJobs, size_t slotBytes, Extent &&extent)
{
  WavePlan p;
  p.perWave = ransac_jobs_per_wave(slotBytes);
  for (int k = 0; k < numJobs; k++)
    if (extent(jobs[k]) > 0) p.live.push_back(k);
  for (size_t q0 = 0; q0 < p.live.size(); q0 += p.perWave) {
    size_t n = 0;
    for (size_t q = q0; q < std::min(p.live.size(), q0 + p.perWave); q++) n += extent(jobs[p.live[q]]);
    p.extent = std::max(p.extent, n);
  }
  return p;
}

// The pinned area of a batch, grown in h: one State per non-empty job (the q-th's at q), then the job table.
template <class State, class Job>
int pinned_states_and_jobs(PinnedBuffer &h, int live, State *&states, Job *&jobs)
{
  Layout L(256);
  L.take((size_t)std::max(live, 1) * sizeof(State));
  int r;
  if ((r = h.grow(L.bytes + (size_t)live * sizeof(Job))) < 0) return r;
  states = h.as<State>();
  jobs = reinterpret_cast<Job *>(h.as<char>() + L.bytes);
  return 0;
}

struct Pipeline;    // extraction, batched and round-1 kernels (pipeline2.h)
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

// Everything a device keeps between calls, one per device index (api.cu: current_ctx()).  Calls use it on its stream:
// like the reference (function-local static caches, cudaSiftH.cu:310,409) the library is single-threaded per device --
// two host threads calling on the same device at the same time would share these buffers.
struct DeviceCtx {
  int dev = -1;
  int sms = 0;                             // multiprocessor count
  cudaStream_t stream = nullptr;           // blocking stream: ordered after legacy default-stream work
  std::map<PipeKey, Pipeline *> pipes;     // batch-of-one pipelines of the drop-in ExtractSift

  // Device buffers grown on demand, and the entry points that use them.  A call may use several at once
  // (cs_match_ratio: knnLists, pairScratch, the tc* tables and knnPartials), so each has its own member.
  GrowBuffer image, points;   // cs_extract_host: the image, the records
  // cs_match_host, cs_match_mutual_host, cs_match_ratio_host, cs_verify_pairs_host: the uploaded sets
  GrowBuffer set1, set2;
  // cs_match_mutual_host, cs_match_ratio_host: the pairs; cs_verify_pairs_host: the input pairs, then the inliers
  GrowBuffer pairs;
  GrowBuffer knnLists;        // cs_match_ratio(_host): both directions' neighbour lists
  GrowBuffer pairScratch;     // cs_match_mutual(_host), cs_match_ratio(_host): ballot words, CTA counts, the total
  GrowBuffer knnPartials;     // cs_match_knn2, cs_match_ratio(_host): the slices of the exact scan
  GrowBuffer verify;          // cs_verify_pairs(_host, _batch), cs_verify_models, cs_verify_essential(_host, _models, _batch)
  GrowBuffer rank;            // cs_rank_records: counters, scratch
  // cs_match_knn2_guided, cs_match_guided(_host, _batch): a wave's tables and headers, and per job its coefficient
  // records, cell grids, sorted candidate copies, knn lists and pair scratch
  GrowBuffer guided;
  PinnedBuffer h_guidedBatch;              // every guided wave's tables (uploaded) and state (copied back)
  // the tensor path (match_tc.cu) of cs_match(_host), cs_match_mutual(_host), cs_match_knn2, cs_match_ratio(_host):
  // operand tiles, B-role copies, row norms, top-3 tables, fallback rows, and 2 x 16 words of flags used alternately
  GrowBuffer tcA, tcB, tcNorms, tcTables, tcRows, tcFlags;
  unsigned long long tcCalls = 0;          // selects the flag area
  bool tcDirty = false;                    // a call returned with an error after it had started to use its flag area
  bool tcConfigured = false;               // the GEMM kernel's shared-memory size is set
  bool tcPendingStats = false;             // h_tcFlags holds the last call's counters, not yet read
  // cs_match_ratio_batch (besides tcA, tcNorms and tcTables): a wave's set, direction and job tables; its neighbour
  // lists and fallback entries; its flags, counters and totals (cleared per wave), then the pair scratch
  GrowBuffer mbTables, mbLists, mbState;
  bool mbConfigured = false;               // the batch GEMM's shared-memory size is set
  PinnedBuffer h_mb;                       // every wave's tables (uploaded) and state (copied back)
  // cs_build_tracks: the statistics, image bases, list table, per-tile totals, per-feature arrays and sort storage
  GrowBuffer tracks;
  PinnedBuffer h_tracks;                   // the statistics (copied back), then the bases and list table
  // cs_triangulate_tracks: the statistics and queue word, the camera table and the spilled members
  GrowBuffer tri;
  PinnedBuffer h_tri;                      // the statistics (copied back), then the camera table
  // cs_absolute_pose_batch, cs_absolute_pose_models: the job table, then a wave's correspondences, slots, slot counts
  // and job states
  GrowBuffer pose;
  PinnedBuffer h_pose;                     // every job's state (copied back), then the job table
  // cs_bundle_adjust: the result words, the trace, the camera, point and observation tables, the camera pieces and
  // partials, the sort storage
  GrowBuffer bundle;
  PinnedBuffer h_bundle;                   // the result words and the trace (copied back), then the camera table
  // cs_rotation_averaging: the result words, the trace, the image and edge tables, the final angles, the incidence
  // sort, the image pieces and partials, the sort storage
  GrowBuffer rotavg;
  // cs_global_positioning: the result words, the trace, the camera, point and observation tables, the pieces, the sorts
  GrowBuffer globalpos;
  PinnedBuffer h_globalpos;                // the result words and the trace (copied back), then the camera table
  PinnedBuffer h_rotavg;                   // the same words, tables and incidences on the host (uploaded, copied back)
  // cs_verify_*: the states a call copies back, and its job table
  PinnedBuffer h_verify;
  // cs_vocab_train: the set table and start draws, the assignments, best scores, sort pairs, word bounds, tile
  // partials and sort storage (cs_vocab_assign uses the batch buffers of cs_match_ratio_batch only)
  GrowBuffer vocab;
  PinnedBuffer h_vocab;                    // the set table and draws (uploaded), the partials and empty-word counts
  // cs_retrieve_pairs: the statistics, image table, keys, postings, inverted file, word and image bounds, idf, the
  // query accumulators of a wave, the candidate pair keys and the cub storage
  GrowBuffer retrieve;
  PinnedBuffer h_retrieve;                 // the statistics (copied back), then the image table
  int retrieveWaves = 0;                   // the waves of the last cs_retrieve_pairs call
  // cs_undistort_images, cs_patch_match_stereo(_geometric), cs_fuse_depth_maps: the image, job and source tables, the per-job
  // counters and the point list's scratch
  GrowBuffer stereo;
  PinnedBuffer h_stereo;                   // the same tables (uploaded), then the counters (copied back)
  // cs_poisson_mesh and cs_simplify_mesh: the result words (copied back); their scratch is allocated and freed per call
  PinnedBuffer h_mesh;

  // pinned host words, allocated by ensure()
  unsigned int *h_counters = nullptr;      // 4: extraction, describe and rank counters
  unsigned int *h_tcFlags = nullptr;       // 16: the tensor path's flag area of the last call
  unsigned int *h_pairTotal = nullptr;     // the pair total of the last mutual or ratio call

  unsigned long long matchStats[4] = {0, 0, 0, 0};
  unsigned long long guidedStats[4] = {0, 0, 0, 0};
  long long verifyStats[8] = {0, 0, 0, 0, -1, 0, 0, 0};
  long long essentialStats[10] = {0, 0, 0, 0, -1, 0, 0, 0, 0, 0};

  int ensure(int d);
  Pipeline *get_pipe(int w, int h, int oct, bool up, float *arena, int *err);
  void drop_pipes(float *arena, bool internalOnly);
};

// CUDASIFT_MATCH_TIMING=1: nine events for timing the kernels of a match or verify call, else null
cudaEvent_t *match_timing_events();
// After the stages' launches: "<header> [us]: name t name t ..." on stderr, stage i timed from tev[i] to tev[i + 1]
// (waits for tev[n]).  header is a printf format.
void report_stage_times(const cudaEvent_t *tev, const char *const *names, int n, const char *header, ...)
    __attribute__((format(printf, 4, 5)));

// ---- matcher ------------------------------------------------------------------------
// the cross-check of a mutual match: pairs with score > minScore and ambiguity < maxAmbiguity, at most maxPairs written
struct MutualArgs {
  float minScore, maxAmbiguity;
  int2 *pairs;
  int maxPairs;
};
int match_exact(SiftPoint *s1, int n1, const SiftPoint *s2, int n2, cudaStream_t st);
// The launchers below run on c.stream.
// tensor path: set 1 against set 2, or with mu (32 or more rows in each set) both directions and then the pairs
int match_tensor(DeviceCtx &c, SiftPoint *s1, int n1, SiftPoint *s2, int n2, const MutualArgs *mu);
bool match_tensor_supported();
void match_tensor_stats(DeviceCtx &c, unsigned long long stats[4]);   // after a synchronize
// cross-check of two finished directions (match_mutual.cu); the total reaches *c.h_pairTotal by the synchronize
int launch_mutual_pairs(DeviceCtx &c, const SiftPoint *s1, int n1, const SiftPoint *s2, int n2, const MutualArgs &mu);
// two nearest neighbours among all candidates (match_knn.cu states the order): idx / score are [n1][2], 8-byte aligned
int knn_exact(DeviceCtx &c, const SiftPoint *s1, int n1, const SiftPoint *s2, int n2, int *idx, float *score);
// tensor path of the same; with idx2 also set 2 against set 1 (match_tc.cu)
int match_knn_tensor(DeviceCtx &c, const SiftPoint *s1, int n1, const SiftPoint *s2, int n2, int *idx1, float *score1,
                     int *idx2, float *score2);
// Lowe's ratio test (COLMAP's rule) on finished knn lists, cross-checked when idx2 != nullptr; the total reaches
// *c.h_pairTotal by the synchronize
struct RatioArgs {
  float maxRatio, maxDistance;
  int2 *pairs;
  int maxPairs;
};
int launch_ratio_pairs(DeviceCtx &c, const int *idx1, const float *score1, int n1, const int *idx2, const float *score2,
                       int n2, const RatioArgs &ra);

// The entry e of a table sorted by a start field (first CTA, first unit) with a[e].*start <= x < a[e + 1].*start;
// every entry spans at least one.
template <class T>
__device__ __forceinline__ int table_find(const T *__restrict__ a, int n, int T::*start, int x)
{
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (a[mid].*start <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---- union-find (tracks.cu, texture.cu) -------------------------------------------------------------------------
// Trees of parent links that keep parent[x] <= x for every x, so each root is the smallest id of its tree whatever the
// order of the threads (DESIGN.md, "Feature tracks", gives the argument).
//
// The root of x with path halving.  Every store writes an ancestor, so parent[x] <= x keeps holding; a store racing
// with another thread's can only leave a different ancestor.
__device__ __forceinline__ int uf_find(int *parent, int x)
{
  volatile int *p = parent;
  int cur = p[x];
  if (cur != x) {
    int prev = x, next;
    while (cur > (next = p[cur])) {
      p[prev] = next;
      prev = cur;
      cur = next;
    }
  }
  return cur;
}

// Joins the trees of u and v (ECL-CC's hook): atomicCAS of the larger root onto the smaller; when the CAS fails, the
// larger root has been hooked meanwhile and the walk continues from the root of the value it read.
__device__ __forceinline__ void uf_link(int *parent, int u, int v)
{
  int ru = uf_find(parent, u), rv = uf_find(parent, v);
  while (ru != rv) {
    const int hi = ru > rv ? ru : rv, lo = ru > rv ? rv : ru;
    const int old = atomicCAS(parent + hi, hi, lo);
    if (old == hi) break;
    if (hi == ru) ru = uf_find(parent, old); else rv = uf_find(parent, old);
  }
}

// One pair list of the flags / write kernels (match_mutual.cu; an ordered list of ordered_list.cuh): the keep test of
// rows [0, n1) of set 1, then pairs {i, jv[i * jstride]} at positions < maxPairs and the total.  A single call passes
// one by value; a batch passes a table in device memory, job k owning the CTAs from cta0 on.
struct PairJob {
  const int *jv; int jstride;
  int n1, n2;
  const int2 *idx1; const float2 *score1;     // ratio: the knn lists of set 1
  const int2 *idx2; const float2 *score2;     // and of set 2 (cross-check), or null
  unsigned int *masks, *blockCounts;          // list_words(n1) ballot words, list_ctas(n1) CTA counts
  int2 *pairs; int maxPairs;
  unsigned int *total;
  int cta0;
};

// ---- batched ratio matching (cs_match_ratio_batch) ------------------------------------------------------------------
// A direction of a wave: the n1 rows of set 1 against the n2 candidates of set 2, with its operand tiles, its units of
// the wave's GEMM, its top-3 table tiles, its resolve CTAs and its neighbour lists.  Built on the host (match_tc.cu).
// A single call's resolve takes one by value: its rows, candidates, norms, max norm, counters and, for the top-2 rule,
// its lists; the table fields stay zero.
struct MbDir {
  const SiftPoint *s1, *s2;
  int n1, n2;
  const float *norms;                 // set 1's row norms
  const float *bmax;                  // set 2's max norm (float bits)
  const unsigned int *bad1, *bad2;    // the sets' bad-input flags: either one gates the direction
  int2 *idx; float2 *score;           // [n1] neighbour lists
  unsigned int *counters;             // [0] fallback rows, [1] groups re-scored, [2] chains
  int aTile0, bTile0;                 // set 1's / set 2's first operand tile
  int n_nt;                           // candidate tiles
  int u0;                             // first GEMM unit (n_mt x n_nt of them)
  int gt0;                            // first table tile (n_mt of them)
  int cta0;                           // first resolve CTA (ceil(n1 / 16) of them)
};
// Where the results of job p of a batch land in pinned memory after the call's synchronize: its pair total and, per
// direction (the second null without the cross-check), the counters and the two sets' bad-input flags.
struct RatioBatchOut {
  const unsigned int *total;
  const unsigned int *counters[2];
  const unsigned int *bad1, *bad2;
};
// Every non-empty job of a batch (argument-checked) in waves on c.stream, without a synchronize; out[p] is filled for
// the non-empty jobs.
int ratio_batch_enqueue(DeviceCtx &c, const cs_match_set *sets, int numSets, const cs_match_job *jobs, int numJobs,
                        float maxRatio, float maxDistance, bool crossCheck, RatioBatchOut *out);
// A wave of knn directions once its four shared launches are in: its jobs (input indices, in order), its pair-job
// table (device) and pair CTAs, and its neighbour lists: the rows of its directions one after the other, rows in all.
struct KnnWave {
  const std::vector<int> &jobs;
  const PairJob *pairJobs;
  int numJobs, pairCtas;
  const int2 *idx;
  const float2 *score;
  int rows;
};
using KnnWaveFinish = std::function<int(const KnnWave &)>;
// The waves of ratio_batch_enqueue with the last step of each wave left to finish (launched on c.stream after the
// exact fallback; name heads the stage timing and lastStage names the step).  ratio_batch_enqueue is this with the
// ratio flags and pair writes.
int knn_batch_enqueue(DeviceCtx &c, const cs_match_set *sets, int numSets, const cs_match_job *jobs, int numJobs,
                      bool crossCheck, RatioBatchOut *out, const char *name, const char *lastStage,
                      const KnnWaveFinish &finish);
// the exact top-2 scan of the rows the wave's resolve listed ({direction, row} entries, *numEntries of them)
int launch_knn_list_fallback(DeviceCtx &c, const MbDir *dirs, const int2 *entries, const unsigned int *numEntries,
                             int cap);
// the ratio flags and pair writes of a wave's jobs (numCtas = the CTAs of all jobs)
int launch_ratio_pairs_batch(DeviceCtx &c, const PairJob *jobs, int numJobs, int numCtas, float maxRatio,
                             float maxDistance);

// The neighbour order of the exact knn searches (match_knn.cu, match_guided.cu): (s, j) comes before (t, k) when the
// score is larger, then the index lower.  The empty entry (0, -1) comes after every positive score and before every
// other one, so non-positive scores never enter.
__device__ __forceinline__ bool knn_before(float s, int j, float t, int k) { return s > t || (s == t && j < k); }

struct Top2 {
  float s1, s2;
  int j1, j2;
};
__device__ __forceinline__ void top2_init(Top2 &t) { t.s1 = t.s2 = 0.0f; t.j1 = t.j2 = -1; }
__device__ __forceinline__ void top2_insert(Top2 &t, float s, int j)
{
  if (knn_before(s, j, t.s1, t.j1)) { t.s2 = t.s1; t.j2 = t.j1; t.s1 = s; t.j1 = j; }
  else if (knn_before(s, j, t.s2, t.j2)) { t.s2 = s; t.j2 = j; }
}

// ---- guided matching (match_guided.cu) ------------------------------------------------------------------------------
// Where job p's results land in pinned memory after the call's synchronize (null for an empty job).
struct GuidedBatchOut {
  const unsigned int *total;
  const unsigned long long *stats;
};
// What a single call (one job) adds: its stage timing is reported as "guided timing n1xn2", and with idx
// (cs_match_knn2_guided, one direction) set 1's lists go to idx / score ([n1][2]) and no pair launches are issued.
struct GuidedSingle {
  int *idx;
  float *score;
};
// Every non-empty job (argument-checked) in waves on c.stream (cs_match_guided_batch, whose header comment states the
// wave rule), without a synchronize; single is null for a batch.
int guided_enqueue(DeviceCtx &c, const cs_match_set *sets, const cs_match_job *jobs, int numJobs, const int *models,
                   const double *models_in, float thresh, float maxRatio, float maxDistance, bool cross,
                   GuidedBatchOut *out, const GuidedSingle *single);

// ---- feature tracks (tracks.cu) ---------------------------------------------------------------------------------
// The kernels of cs_build_tracks (argument-checked, at least one pair in all) on c.stream, without a synchronize; the
// eight statistics reach c.h_tracks (unsigned long long) by the caller's synchronize.
int tracks_enqueue(DeviceCtx &c, const int *imageSizes, int numImages, const cs_track_list *lists, int numLists,
                   int minLength, bool drop, int *trackOf, int *offsets, int maxTracks, int *members, int maxMembers);

// ---- vocabulary and retrieval (vocab.cu) ------------------------------------------------------------------------
// One assignment call: the sets with the vocabulary appended, the jobs (a, vocabulary), each set's first global id,
// where each job's counters land (RatioBatchOut) and the waves run.
struct VocabAssign {
  std::vector<cs_match_set> sets;
  std::vector<cs_match_job> jobs;
  std::vector<int> base;
  std::vector<RatioBatchOut> out;
  int waves = 0;
};
// The waves of cs_vocab_assign (argument-checked) on c.stream, without a synchronize: wordOf[base_a + i] = j1 of row i
// of set a, and with best its score.
int vocab_assign_enqueue(DeviceCtx &c, const cs_match_set *sets, int numSets, const void *vocab, int numWords,
                         int *wordOf, float *best, VocabAssign &va);
// after the synchronize: groups re-scored, exact chains, fallback rows, gated sets, waves
void vocab_assign_stats(const VocabAssign &va, unsigned long long st[5]);
// The start draws of cs_vocab_train (host): the first numWords distinct indices of the counter-based generator.
std::vector<int> vocab_start_draws(unsigned long long seed, int M, int numWords);
// cs_vocab_train (argument-checked), synchronizing once per iteration; trace [maxIterations][4] is written whole.
// Returns the iterations run.
int vocab_train(DeviceCtx &c, const cs_match_set *sets, int numSets, int numWords, int maxIterations,
                unsigned long long seed, SiftPoint *vocab, double *trace, long long stats[4]);
// cs_retrieve_pairs (argument-checked, some feature) on c.stream, without a synchronize; the seven statistics reach
// c.h_retrieve (unsigned long long) by the caller's synchronize, the wave count c.retrieveWaves.
int retrieve_queries_per_wave(int numImages);
int retrieve_enqueue(DeviceCtx &c, const int *imageSizes, int numImages, const int *wordOf, int numWords, int topK,
                     int *neighbours, double *scores, double *idf, int *pairs, int maxPairs);

// ---- triangulation (triangulate.cu) -----------------------------------------------------------------------------
// The launch of cs_triangulate_tracks (argument-checked, numTracks > 0) on c.stream, without a synchronize; the eight
// statistics reach c.h_tri (unsigned long long) by the caller's synchronize.
int triangulate_enqueue(DeviceCtx &c, const cs_match_set *sets, int numImages, const double *Ks, const double *Rs,
                        const double *ts, const int *offsets, int numTracks, const int *members, int numMembers,
                        int numTrials, double maxError, double minTriAngle, unsigned long long seed, double *points,
                        int *counts, float *errors, unsigned char *inlier);

// ---- absolute pose (pose.cu) ------------------------------------------------------------------------------------
// The waves of an argument-checked batch on c.stream, without a synchronize: with full the five launches per wave, else
// the first three (gather, hypotheses, scoring; the slots of the last wave stay in c.pose).  The q-th non-empty job's
// state reaches c.h_pose by the caller's synchronize.
int pose_enqueue(DeviceCtx &c, const double *points, int numPoints, const cs_pose_job *jobs, int numJobs,
                 const double *Ks, int numLoops, double maxError, bool full);
// after a full enqueue and a synchronize: the q-th non-empty job's pose, statistics and count
int pose_result(const DeviceCtx &c, int q, double R[9], double t[3], long long stats[8]);
// after an enqueue of one job without full: every slot's R, t (NaN-filled when empty) and count (synchronizes);
// returns the job's number of valid correspondences
int pose_models_to_host(DeviceCtx &c, const cs_pose_job &job, int numLoops, double *h_R, double *h_t, int *h_counts);

// ---- bundle adjustment (bundle.cu) -----------------------------------------------------------------------------
// The camera block of a call: 9 when an image refines an intrinsic or has a nonzero distortion coefficient, else 6.
int bundle_camera_block(int numImages, const double *dists, const unsigned char *refine);
// The launches of cs_bundle_adjust_intrinsics (argument-checked, numTracks > 0) on c.stream, without a synchronize;
// the results reach c.h_bundle by the caller's synchronize, and bundle_result reads them.
int bundle_enqueue(DeviceCtx &c, const cs_match_set *sets, int numImages, const double *Ks, const double *dists,
                   const unsigned char *refine, int loss, double lossScale, const double *Rs, const double *ts,
                   const unsigned char *fixed, const int *offsets, int numTracks, const int *members, int numMembers,
                   const unsigned char *use, double *points, int maxIterations, int maxLinearIterations,
                   double linearTol, double maxError, float *errors, unsigned char *inlier);
// after the synchronize, for the camera block nc the call ran: the final K, (k1, k2) (nc == 9 only; either may be
// NULL), R, t of every image, the costs, the trace (may be NULL) and the statistics; returns the number of accepted
// steps
int bundle_result(const DeviceCtx &c, int nc, int numImages, int maxIterations, double *K_out, double *dist_out,
                  double *R_out, double *t_out, double cost[2], double *trace, long long stats[8]);
// The launch of cs_undistort_records (argument-checked, at least one record) on c.stream, without a synchronize.
int undistort_enqueue(DeviceCtx &c, const cs_match_set *sets, int numImages, const double *Ks, const double *dists,
                      void *const *d_out);

// ---- rotation averaging (rotavg.cu) -------------------------------------------------------------------------------
// The host part of cs_rotation_averaging (argument-checked, numEdges > 0): the spanning tree, the start rotations and
// the image, edge and incidence tables in c.h_rotavg.
int rotavg_prepare(DeviceCtx &c, int numImages, const int *edges, int numEdges, const double *Rrel,
                   const double *weights, int refImage, int maxIterations);
// After rotavg_prepare: the sort and the cooperative launch on c.stream, without a synchronize; the results reach
// c.h_rotavg by the caller's synchronize, and rotavg_result reads them.
int rotavg_enqueue(DeviceCtx &c, int numImages, int numEdges, int maxIterations, int maxLinearIterations,
                   double linearTol, double sigmaDeg);
// after the synchronize: R_out, the residual angles and inlier bytes (either may be NULL), the costs, the trace (may be
// NULL) and the statistics (may be NULL); returns the IRLS iterations run
int rotavg_result(const DeviceCtx &c, int numImages, int numEdges, int maxIterations, double maxAngleDeg,
                  double *R_out, double *residuals, unsigned char *inlier, double cost[2], double *trace,
                  long long stats[6]);

// ---- global positioning (globalpos.cu) -------------------------------------------------------------------------------
// The launches of cs_global_positioning (argument-checked, numTracks > 0) on c.stream, without a synchronize; the results
// reach c.h_globalpos by the caller's synchronize, and globalpos_result reads them.
int globalpos_enqueue(DeviceCtx &c, const cs_match_set *sets, int numImages, const double *Ks, const double *Rs,
                      const int *offsets, int numTracks, const int *members, int numMembers, const unsigned char *use,
                      int refImage, unsigned long long seed, int loss, double lossScale, int maxIterations,
                      int maxLinearIterations, double linearTol, double *points);
// after the synchronize: t_out, the costs, the trace (may be NULL) and the statistics (may be NULL); returns the
// accepted steps
int globalpos_result(const DeviceCtx &c, int numImages, const double *Rs, int maxIterations, double *t_out,
                     double cost[2], double *trace, long long stats[8]);

// ---- dense reconstruction (stereo.cu) -----------------------------------------------------------------------------
// The launch of cs_undistort_images (argument-checked, numImages > 0) on c.stream, without a synchronize; the outside
// counts reach *outside (pinned, numImages of them) by the caller's synchronize.
int undistort_images_enqueue(DeviceCtx &c, const cs_image *images, int numImages, const double *Ks,
                             const double *dists, float *const *out, const unsigned long long **outside);
// The launches of cs_patch_match_stereo (argument-checked, numJobs > 0) on c.stream, without a synchronize; per job
// the counters {0, invalid view evaluations, pixels of final cost 2} reach *counts (pinned, 3 per job) by the caller's
// synchronize.
int patch_match_enqueue(DeviceCtx &c, const cs_image *images, int numImages, const double *Ks, const double *Rs,
                        const double *ts, const cs_stereo_job *jobs, int numJobs, int radius, int step,
                        int numIterations, int topK, unsigned long long seed, const unsigned long long **counts);
// The launches of cs_patch_match_stereo_geometric (argument-checked, numJobs > 0) on c.stream, without a synchronize;
// per job the counters {0, invalid view evaluations, pixels of final cost >= 2}, then per job {valid view evaluations
// capped at geomMaxError, pixels started from a draw, 0} reach *counts (pinned, 6 per job) by the caller's synchronize.
int patch_match_geometric_enqueue(DeviceCtx &c, const cs_image *images, int numImages, const double *Ks,
                                  const double *Rs, const double *ts, const cs_depth_prior *priors,
                                  const cs_stereo_job *jobs, int numJobs, int radius, int step, int numIterations,
                                  int topK, double geomWeight, double geomMaxError, unsigned long long seed,
                                  const unsigned long long **counts);
// The launches of cs_fuse_depth_maps (argument-checked, numJobs > 0) on c.stream, without a synchronize; the point
// total reaches **total (pinned) by the caller's synchronize.
int fuse_enqueue(DeviceCtx &c, const cs_image *images, int numImages, const double *Ks, const double *Rs,
                 const double *ts, const cs_stereo_job *jobs, int numJobs, float maxCost, int minConsistent,
                 double maxReprojError, double maxDepthError, double maxNormalErrorDeg, float *xyz, float *normal,
                 float *intensity, int *source, int maxPoints, unsigned int **total);

// ---- Poisson meshing (mesh.cu) -------------------------------------------------------------------------------------
// The launches of cs_poisson_mesh (pointWeight 0) or cs_poisson_mesh_screened (pointWeight > 0), argument-checked, on
// st, with the scratch allocated and freed on st, without a synchronize; the result words (mesh_result_bytes of them)
// reach h_result (pinned) by the caller's synchronize.
int mesh_run(const float *xyz, const float *normal, const float *intensity, int numPoints, int depth, double scale,
             double pointWeight, int maxIterations, double tol, double trim, float *vertices, float *vertexIntensity,
             int maxVertices, int *triangles, int maxTriangles, float *chiOut, cudaStream_t st, void *h_result);
size_t mesh_result_bytes();
// after the synchronize: info_out ([7], or [8] when screened) and stats_out (either may be NULL); returns the full
// triangle count
int mesh_result(const void *h_result, int numPoints, int maxVertices, int maxTriangles, bool screened, double *info,
                long long stats[10]);

// ---- mesh simplification (simplify.cu) -----------------------------------------------------------------------------
// cs_simplify_mesh after its argument checks, on st with per-pass readbacks through h_result (pinned,
// simplify_result_bytes), the scratch allocated and freed on st; fills info (may be NULL) and stats (may be NULL) and
// returns the full triangle count.
int simplify_run(const float *vertices, const float *intensity, int numVertices, const int *triangles, int numTriangles,
                 int targetTriangles, double maxError, double boundaryWeight, float *outVertices, float *outIntensity,
                 int maxOutVertices, int *outTriangles, int maxOutTriangles, cudaStream_t st, void *h_result,
                 double *info, long long *stats);
size_t simplify_result_bytes();

// ---- mesh cleaning (clean.cu) ----------------------------------------------------------------------------------------
// cs_clean_mesh after its argument checks (numTriangles > 0), on st with readbacks through h_result (pinned,
// clean_result_bytes), the scratch allocated and freed on st; fills info (may be NULL; 3 entries) and stats (may be
// NULL; 19 entries) and returns the full triangle count.
int clean_run(const float *vertices, const float *intensity, int numVertices, const int *triangles, int numTriangles,
              int removeDegenerate, double longEdgeFactor, int removeNonManifold, int minComponentFaces,
              double minComponentFraction, int maxHoleEdges, int smoothIterations, double lambda, double mu,
              float *outVertices, float *outIntensity, int maxOutVertices, int *outTriangles, int maxOutTriangles,
              cudaStream_t st, void *h_result, double *info, long long *stats);
size_t clean_result_bytes();

// ---- mesh texturing (texture.cu) -----------------------------------------------------------------------------------
// The depth-buffer bytes of one image group (cs_set_tuning("texture_group_bytes"); 0 or less: 1 GiB).
extern long long g_texture_group_bytes;
// cs_texture_mesh_photo's view selection: the data term (0 area, 1 GMI) and the outlier test (outlierK 0: off).
struct TexturePhoto {
  int dataTerm;
  double outlierK, outlierMinSigma;
};
// cs_texture_mesh (photo NULL), cs_texture_mesh_photo and cs_texture_mesh_bp (maxBpSweeps >= 0, with photo) after
// their argument checks (numTriangles > 0), on st with readbacks through h_result (pinned, texture_result_bytes), the
// scratch allocated and freed on st; fills charts_out, info (may be NULL; 2 entries, 3 with BP) and stats (may be NULL;
// 11 entries, 16 with photo, 20 with BP) and returns the full chart count.
int texture_run(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
                const float *vertices, int numVertices, const int *triangles, int numTriangles, double lambda,
                double maxViewAngleDeg, double depthTol, int padding, int atlasWidth, int maxSweeps, float *atlas,
                int maxAtlasRows, float *uv, int *faceView, int *faceChart, int *chartsOut, int maxCharts,
                cudaStream_t st, void *h_result, double *info, long long *stats, const TexturePhoto *photo = nullptr,
                int maxBpSweeps = -1);
size_t texture_result_bytes();

// ---- seam levelling (seams.cu) -------------------------------------------------------------------------------------
// cs_level_texture_seams after its argument checks, on st with readbacks through h_result (pinned,
// seams_result_bytes), the scratch allocated and freed on st; fills info (may be NULL) and stats (may be NULL) and
// returns the unknown count (0 for invalid input).
int seams_run(const float *vertices, int numVertices, const int *triangles, int numTriangles, const int *faceView,
              const float *uv, const int *charts, int numCharts, const float *atlas, int atlasRows, int atlasWidth,
              int padding, double smoothness, double regularization, int maxIterations, double tol, float *outAtlas,
              float *cornerOffset, cudaStream_t st, void *h_result, double *info, long long *stats);
size_t seams_result_bytes();
// cs_level_texture_seams_local after its argument checks, likewise (h_result pinned, seams_local_result_bytes); returns
// the free-texel count (0 for invalid input).
int seams_local_run(const float *vertices, int numVertices, const int *triangles, int numTriangles,
                    const int *faceView, const float *uv, const int *charts, int numCharts, const float *atlas,
                    int atlasRows, int atlasWidth, int padding, int stripWidth, int maxIterations, double tol,
                    float *outAtlas, cudaStream_t st, void *h_result, double *info, long long *stats);
size_t seams_local_result_bytes();

// ---- photometric mesh refinement (refine.cu) -----------------------------------------------------------------------
// cs_mesh_refine after its argument checks (numTriangles > 0), on st with readbacks through h_result (pinned,
// refine_result_bytes), the scratch allocated and freed on st; writes outVertices, fills info (may be NULL; 4 entries)
// and stats (may be NULL; 8 entries) and returns the status.
int refine_run(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
               const float *vertices, int numVertices, const int *triangles, int numTriangles, const int *pairs,
               int numPairs, int windowRadius, double smoothness, double step, int maxIterations, double depthTol,
               float *outVertices, cudaStream_t st, void *h_result, double *info, long long *stats);
size_t refine_result_bytes();

// ---- geometric verification (verify.cu) -------------------------------------------------------------------------
// The model id verify_enqueue uses for cs_verify_essential (not a model value of the public cs_verify_pairs).
#define VERIFY_ESSENTIAL 3
// The intrinsics of an essential call (row-major, checked by the caller).
struct VerifyCalib {
  double K1[9], K2[9];
};
// The waves of an argument-checked batch (one job for a single call) on c.stream, without a synchronize: per wave steps
// 1-4, and with full also 5-8 (arg-max, refit, output; without full the slots of the last wave stay in c.verify).  The
// q-th non-empty job's state reaches c.h_verify by the caller's synchronize.  cal (numJobs entries) is read for
// VERIFY_ESSENTIAL only.
int verify_enqueue(DeviceCtx &c, const cs_verify_job *jobs, int numJobs, const VerifyCalib *cal, int model, int numLoops,
                   float thresh, bool full);
// after a full enqueue and a synchronize: the q-th non-empty job's inlier count, pixel model and statistics
int verify_result(const DeviceCtx &c, int q, int numPairs, double model_out[9], long long stats[8]);
// the same after a full VERIFY_ESSENTIAL enqueue: E, R, t and the ten statistics of cs_verify_essential_stats
int verify_essential_result(const DeviceCtx &c, int q, int numPairs, double E[9], double R[9], double t[3],
                            long long stats[10]);
// after an enqueue of one job without full: every slot's pixel model (E for VERIFY_ESSENTIAL), count and the
// normalisation (synchronizes); returns numValid
int verify_models_to_host(DeviceCtx &c, const cs_verify_job &job, int numLoops, int model, const VerifyCalib *cal,
                          double *h_models, int *h_counts, double h_norm[5]);

inline int idivup(int a, int b) { return (a + b - 1) / b; }
inline int ialignup(int a, int b) { return (a % b != 0) ? (a - a % b + b) : a; }

}  // namespace cs
