/*
 * cudasift_b200.h -- C ABI of libcudasift_b200.so (plain pointers and sizes only).
 *
 * The reference (Celebrandil/CudaSift) has no FFI: its boundary is the C++ header pair
 * cudaSift.h / cudaImage.h, which this library also exports with identical mangled
 * symbols (include/cudaSift.h, include/cudaImage.h).  This header is the additive
 * `extern "C"` surface a binding (ctypes, cgo, JNI ...) would use; every entry point
 * names the reference interface it stands for.  See INTEGRATION.md for the binding stubs.
 *
 * Conventions: functions returning int return >= 0 on success and a negative CS_E_* code
 * on failure (cs_last_error() has the text).  Device pointers are raw CUDA device
 * addresses in the current device's address space.  SiftPoint records are the 576-byte
 * layout of cudaSift.h:6-22.  All calls are synchronous unless named *_submit.
 */
#ifndef CUDASIFT_B200_H
#define CUDASIFT_B200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CS_E_CUDA     (-1)   /* a CUDA runtime call failed */
#define CS_E_ARG      (-2)   /* invalid argument */
#define CS_E_NOMEM    (-3)
#define CS_E_NODEV    (-4)   /* no CUDA device: the product has no CPU fallback */

const char *cs_last_error(void);
const char *cs_version(void);

/* InitCuda (cudaSiftH.cu:19-37).  Returns the device index actually selected. */
int cs_init(int device);
/* Number of kernels this library has launched so far in this process. */
unsigned long long cs_launch_count(void);
/* Tuning hook (benchmarks and tests only).  Keys: "legacy" (1 = the round-1 per-image kernels for pipelines
 * created afterwards, 0 = the batched TMA pipeline), "cap32" (0 = do not reproduce the reference's cap of 32
 * extrema per 30x8 block and scale, cudaSiftD.cu:1371), "d2_hs" / "pa_rows" (rows per detector stream / per CTA
 * of the first pyramid kernel, 0 = automatic), "sd_split" (0 = every ScaleDown of a batch in the chain kernel),
 * "cap32_limit" (the cap's limit, 1..199; default 32).  Returns 0, or CS_E_ARG for an unknown key. */
int cs_set_tuning(const char *key, int value);
/* Number of launches one steady-state cs_extractor_submit_* / cs_match issues. */
int cs_extract_launches_per_image(int numOctaves, int scaleUp);

/* ---- raw device memory helpers (for bindings without a CUDA allocator) ---- */
void *cs_device_alloc(size_t bytes);
int cs_device_free(void *d_ptr);
int cs_memcpy_h2d(void *d_dst, const void *h_src, size_t bytes);
int cs_memcpy_d2h(void *h_dst, const void *d_src, size_t bytes);
int cs_memset_d(void *d_dst, int value, size_t bytes);
void *cs_host_alloc_pinned(size_t bytes);
int cs_host_free_pinned(void *h_ptr);
int cs_device_sync(void);

/* AllocSiftTempMemory / FreeSiftTempMemory (cudaSiftH.cu:39-70). */
float *cs_alloc_temp(int width, int height, int numOctaves, int scaleUp);
int cs_free_temp(float *d_tmp);
size_t cs_temp_floats(int width, int height, int numOctaves, int scaleUp);

/* ExtractSift (cudaSiftH.cu:72-144) on a device-resident float image (row stride
 * `pitch` floats).  d_pts: device array of maxPts records (required).  h_pts: optional
 * host array that receives the first numPts records.  d_tmp: optional arena from
 * cs_alloc_temp (NULL = internal, cached).  Returns numPts. */
int cs_extract(const float *d_img, int width, int height, int pitch, int numOctaves,
               double initBlur, float thresh, float lowestScale, int scaleUp,
               float *d_tmp, void *d_pts, void *h_pts, int maxPts);

/* CudaImage::Download + ExtractSift with host buffers: h_img is width*height packed
 * floats; h_pts receives the records.  Host<->device copies happen inside. */
int cs_extract_host(const float *h_img, int width, int height, int numOctaves,
                    double initBlur, float thresh, float lowestScale, int scaleUp,
                    void *h_pts, int maxPts);

/* MatchSiftData (matching.cu:1090-1206): fills score/ambiguity/match/match_xpos/
 * match_ypos of set 1 on the device; if h_s1 != NULL the same 5 fields are copied into
 * the host records (matching.cu:1195-1199).  mode: 0 = auto, 1 = exact FP32 SIMT path,
 * 2 = wgmma tensor-core path (+ exact FP32 re-score).  Returns 0; *ms gets the time. */
int cs_match(void *d_s1, int n1, void *d_s2, int n2, void *h_s1, int mode, double *ms);
/* Same with host record arrays (copies both sets up, matches, copies 5 fields back). */
int cs_match_host(void *h_s1, int n1, const void *h_s2, int n2, int mode, double *ms);
/* Statistics of the last tensor-core match on this thread's device:
 * out[0]=candidate groups emitted, out[1]=groups re-scored, out[2]=(row,partition)
 * pairs that took the exact-scan fallback, out[3]=path used (1 or 2). */
int cs_match_stats(unsigned long long out[4]);

/* FindHomography (matching.cu:1000-1087): RANSAC over the matches of set 1.  homography: 9 floats
 * (row-major 3x3, [8] = 1).  Samples are drawn with rand(): srand() beforehand for repeatability. */
int cs_find_homography(void *d_pts, int numPts, float *homography, int *numMatches, int numLoops,
                       float minScore, float maxAmbiguity, float thresh, double *ms);

/* ImproveHomography (geomFuncs.cpp:6-72): host-side iterated least-squares refinement over the
 * HOST records (the reference runs it on data.h_data with OpenCV); fills match_error of every
 * record and overwrites homography[0..8]; *numFit = matches within thresh. */
int cs_improve_homography(void *h_pts, int numPts, float *homography, int numLoops, float minScore,
                          float maxAmbiguity, float thresh, int *numFit);

/* ---- stage-level entry points (reference: cudaSiftH.h:11-22), used by parity tests ---- */
int cs_lowpass(const float *d_src, float *d_dst, int width, int height, int pitch, float sigma);
int cs_scaledown(const float *d_src, float *d_dst, int width, int height, int pitch, int newpitch);
int cs_scaleup(const float *d_src, float *d_dst, int width, int height, int pitch, int newpitch);
/* PrepareLaplaceKernels (cudaSiftH.cu:439-458): kernel[8*12*16] on the host. */
int cs_laplace_taps(int numOctaves, float initBlur, float *h_kernel);
/* LaplaceMulti (cudaSiftH.cu:460-487): materialises the 7 DoG planes (plane stride
 * height*pitch floats) with the same device code the fused detector uses. */
int cs_dog_planes(const float *d_base, float *d_dog, int width, int height, int pitch,
                  int numOctaves, int octave);
/* Hardware bilinear fetches as the gather stages see them (texture set-up of
 * cudaSiftH.cu:186-205): out[i] = tex2D(img, xs[i], ys[i]); all pointers device. */
int cs_tex_probe(const float *d_img, int width, int height, int pitch,
                 const float *d_xs, const float *d_ys, int n, float *d_out);

/* ---- pipelined extractor (extension; the reference API is strictly synchronous) ----
 * One extractor = one CUDA stream + arena + SiftPoint array + pinned staging.  Several
 * extractors on one device overlap their images; one process per GPU shards a batch. */
typedef struct cs_extractor cs_extractor;
cs_extractor *cs_extractor_create(int width, int height, int numOctaves, int maxPts, int scaleUp);
int cs_extractor_destroy(cs_extractor *ex);
/* Enqueue ExtractSift of a device image on the extractor's stream; returns at once. */
int cs_extractor_submit_device(cs_extractor *ex, const float *d_img, int pitch,
                               double initBlur, float thresh, float lowestScale);
/* Enqueue H2D copy (from pinned or pageable host memory) + ExtractSift + D2H of the
 * count and records into the extractor's pinned result buffer. */
int cs_extractor_submit_host(cs_extractor *ex, const float *h_img,
                             double initBlur, float thresh, float lowestScale);
/* Same for an 8-bit greyscale image (width*height bytes, packed): 4x less PCIe traffic; the
 * conversion to float on the device is exact, so results equal submit_host of the float image. */
int cs_extractor_submit_host_u8(cs_extractor *ex, const unsigned char *h_img,
                                double initBlur, float thresh, float lowestScale);
/* One image, synchronously, with CUDA events at the stage boundaries of the extractor's
 * stream: out_ms = {LowPass (+ first ScaleDown), ScaleDown chain, detect (blur+DoG+extrema), describe
 * (orientation+descriptor), total}.  Returns numPts. */
int cs_extractor_profile(cs_extractor *ex, const float *d_img, int pitch, double initBlur,
                         float thresh, float lowestScale, float out_ms[5]);
/* Wait for the last submit; returns numPts. */
int cs_extractor_wait(cs_extractor *ex);

/* ---- batched extraction: what replaces the caller's loop over images (mainSift.cpp:65-69) ----
 * One submit runs every stage ONCE for up to `batch` images of the same size: the pyramid, the detector
 * (all octaves of all images) and the descriptor kernel each see the whole batch in one launch.
 * cs_max_batch() = the largest batch one extractor takes.  Image i uses record slot i (maxPts records each). */
int cs_max_batch(void);
cs_extractor *cs_extractor_create_batch(int width, int height, int numOctaves, int maxPts, int scaleUp, int batch);
/* d_imgs: n device images (16-byte aligned, common pitch, a multiple of 4 floats). */
int cs_extractor_submit_device_batch(cs_extractor *ex, int n, const float *const *d_imgs, int pitch,
                                     double initBlur, float thresh, float lowestScale);
/* h_imgs: n host images of width*height packed floats; copies are enqueued on the extractor's stream. */
int cs_extractor_submit_host_batch(cs_extractor *ex, int n, const float *const *h_imgs,
                                   double initBlur, float thresh, float lowestScale);
/* Wait for the last submit: counts[i] = numPts of image i (counts may be NULL); after a host submit the records
 * of every image are in its pinned slot (cs_extractor_host_points_at).  Returns the sum of the counts. */
int cs_extractor_wait_batch(cs_extractor *ex, int *counts);
int cs_extractor_count(cs_extractor *ex, int slot);
void *cs_extractor_device_points_at(cs_extractor *ex, int slot);
void *cs_extractor_host_points_at(cs_extractor *ex, int slot);
float *cs_extractor_host_image_at(cs_extractor *ex, int slot);
/* ---- ranked batch extraction: a fixed feature budget per image, in a fixed order ----
 * Each image's slot receives the min(maxPts, found) records with the largest |sharpness|, sorted by the rank key
 * (|sharpness| descending, then subsampling, ypos, xpos, scale, orientation ascending; numpy:
 * lexsort((orientation, scale, xpos, ypos, subsampling, -abs(sharpness)))).  They are, byte for byte, the first
 * maxPts records of a plain extractor's output (maxPts = maxCandidates) sorted by that key, whatever order the
 * detector's atomics left them in.  The pipeline writes up to maxCandidates records per image into a candidate area;
 * the ranking stage selects on the device and only the output records cross PCIe after a host submit.
 * Requires 1 <= maxPts <= maxCandidates <= 262144 and the batched pipeline (not cs_set_tuning("legacy", 1));
 * otherwise returns NULL and cs_last_error() names the invalid argument (CS_E_ARG), before any CUDA call.
 * maxPts == maxCandidates returns every record in the fixed order.  cs_extractor_wait_batch returns the ranked
 * counts; cs_extractor_device_points_at / host_points_at address the output slots. */
cs_extractor *cs_extractor_create_ranked(int width, int height, int numOctaves, int maxPts, int scaleUp, int batch,
                                         int maxCandidates);
/* Records found for image `slot` in the last wait (ranked: in the candidate area).  A value equal to maxCandidates
 * means the candidate area overflowed: the output is still sorted, but it is a subset that may depend on atomic
 * order rather than the strongest maxPts records. */
int cs_extractor_candidates(cs_extractor *ex, int slot);
/* The ranking stage on its own: d_out (device, must not overlap d_in) receives the min(n, maxOut) records of d_in
 * (n device records) with the smallest rank key, in key order.  Synchronous; returns the number written. */
int cs_rank_records(const void *d_in, int n, void *d_out, int maxOut);
/* Stage times of one batch (see cs_extractor_profile); returns the sum of the counts.  For a ranked extractor the
 * total (out_ms[4]) includes the ranking stage, which runs after describe: ranking = total - out_ms[0..3]. */
int cs_extractor_profile_batch(cs_extractor *ex, int n, const float *const *d_imgs, int pitch, double initBlur,
                               float thresh, float lowestScale, float out_ms[5]);
/* Host logic of the batched detector (no device needed; tests): its work list for n images -- per item 4 ints
 * {level | image << 8, first column, first tested row, rows per row stream}; a strip tests 244 columns
 * (first column + 1 ...), an item two streams of rows.  Returns the number of items (out holds capItems). */
int cs_detector_items(int width, int height, int numOctaves, int scaleUp, int n, int hs, unsigned int *out, int capItems);
/* Parity tests: pyramid level `level` of image slot `slot` as left by the last submit, packed into h_out
 * (may be NULL); returns width | height << 16 of that level. */
int cs_extractor_read_level(cs_extractor *ex, int slot, int level, float *h_out);
void *cs_extractor_device_points(cs_extractor *ex);
/* After a submit_host + wait: pointer to the pinned host records. */
void *cs_extractor_host_points(cs_extractor *ex);
/* Pinned host staging image of the extractor (width*height floats), for zero-copy fills. */
float *cs_extractor_host_image(cs_extractor *ex);

/* ---- device timers: CUDA events recorded on an extractor's stream (NULL = legacy
 * default stream); cs_event_elapsed_ms waits for `b`. ---- */
void *cs_event_create(void);
int cs_event_destroy(void *ev);
int cs_event_record(void *ev, cs_extractor *ex);
double cs_event_elapsed_ms(void *a, void *b);

#ifdef __cplusplus
}
#endif
#endif
