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
 * pairs that took the exact-scan fallback, out[3]=path used (1 or 2).  After a mutual
 * match, out[0..2] are both directions summed. */
int cs_match_stats(unsigned long long out[4]);

/* Mutual (cross-checked) nearest-neighbour matching, both directions in one call.
 * - Set 1's score/ambiguity/match/match_xpos/match_ypos are written exactly as cs_match(s1, n1, s2, n2) writes
 *   them, and set 2's exactly as cs_match(s2, n2, s1, n1) does, bit for bit (including quirk Q7: the reverse
 *   direction only visits the set-1 rows below 32*floor(n1/32)).  Descriptors and all other fields are untouched.
 * - The pairs are the (i, j) with s1[i].match == j >= 0, s2[j].match == i, s1[i].score > minScore and
 *   s1[i].ambiguity < maxAmbiguity (strict, as cs_find_homography), stored as int pairs {i, j} in increasing i.
 *   Each j appears at most once, so there are at most min(n1, n2).  The order does not depend on atomics.
 * - mode as for cs_match; auto (0) picks the tensor path when both sets have 256 records or more.  The two sets are
 *   converted for the tensor cores once, for both directions.
 * - n1 == 0 or n2 == 0 returns 0 and writes nothing.  *ms (may be NULL) gets the event time of the whole call.
 * Returns the number of mutual pairs (only the first maxPairs are written to d_pairs, device, 8-byte aligned), or
 * CS_E_*.  CS_E_ARG, before any CUDA call, for n < 0, a NULL set with n > 0, maxPairs < 0, NULL pairs with
 * maxPairs > 0, mode not in {0, 1, 2} and overlapping set-1 and set-2 record ranges. */
int cs_match_mutual(void *d_s1, int n1, void *d_s2, int n2, float minScore, float maxAmbiguity,
                    int *d_pairs, int maxPairs, int mode, double *ms);
/* Same with host record arrays and a host pairs buffer: copies both sets up, matches, and copies the five match
 * fields of both sets and the first min(total, maxPairs) pairs back. */
int cs_match_mutual_host(void *h_s1, int n1, void *h_s2, int n2, float minScore, float maxAmbiguity,
                         int *h_pairs, int maxPairs, int mode, double *ms);

/* Two nearest neighbours: for every row i of set 1, among ALL n2 rows of set 2 (no quirk Q7 tail), with the reference's
 * score (the sequential k = 0..127 FMA chain, the value MatchSiftData writes) and only scores > 0 counted:
 *   j1 = the lowest index with the largest score, j2 = the lowest index != j1 with the largest remaining score (it may
 *   equal score1); a missing neighbour is index -1 with score 0.0f.
 * d_idx[i][0..1] = {j1, j2}, d_score[i][0..1] = {score1, score2} (device, [n1][2] each, 8-byte aligned).  The records
 * are only read, so the sets may overlap (a set against itself).  mode: 0 = auto (tensor path on sm_90 when n1 and n2
 * are >= 256), 1 = exact FP32 SIMT path, 2 = tensor path (any size); both give the same bits.  n1 == 0 or n2 == 0
 * returns 0 and writes nothing.  Returns 0 or CS_E_*; CS_E_ARG, before any CUDA call, for n < 0, a NULL set with
 * n > 0, NULL idx / score with n1 > 0, mode not in {0, 1, 2}, output buffers that are not 8-byte aligned or that
 * overlap a record range or each other.  cs_match_stats reports the call. */
int cs_match_knn2(const void *d_s1, int n1, const void *d_s2, int n2, int *d_idx, float *d_score, int mode, double *ms);
/* Lowe's ratio test on the two nearest neighbours (COLMAP's max_ratio / max_distance / cross_check):
 * d = acos(min(score, 1)) in double, and (i, j1) is kept when j1 >= 0, d1 <= maxDistance and d1 < maxRatio * d2
 * (a missing second neighbour gives d2 = pi / 2).  crossCheck != 0: also set 2 against set 1, and (i, j) is kept only
 * if row j of set 2 passes the same test and its j1 is i (the auto mode then needs 256 rows in both sets).  Pairs are
 * int pairs {i, j} in increasing i (with crossCheck each j at most once); the order depends only on the values.
 * Returns the number of pairs and writes the first maxPairs (device, 8-byte aligned), or CS_E_*: CS_E_ARG as for
 * cs_match_knn2, and for maxPairs < 0, NULL pairs with maxPairs > 0 and a NaN maxRatio or maxDistance.  The knn lists
 * live in per-device scratch.  With crossCheck, cs_match_stats reports both directions summed. */
int cs_match_ratio(const void *d_s1, int n1, const void *d_s2, int n2, float maxRatio, float maxDistance, int crossCheck,
                   int *d_pairs, int maxPairs, int mode, double *ms);
/* Same with host record arrays and a host pairs buffer. */
int cs_match_ratio_host(const void *h_s1, int n1, const void *h_s2, int n2, float maxRatio, float maxDistance,
                        int crossCheck, int *h_pairs, int maxPairs, int mode, double *ms);

/* Geometric verification of a correspondence list (RANSAC on the device), for any int pair list {i, j} such as
 * cs_match_mutual and cs_match_ratio write.  Pair k, {i, j} = d_pairs[2k..2k+1], is (s1[i].xpos, s1[i].ypos) <->
 * (s2[j].xpos, s2[j].ypos).  A pair is invalid when i is outside [0, n1), j outside [0, n2) or one of its four coordinates
 * is not finite; invalid pairs are never sampled and never inliers.  The records are only read.
 * - model: CS_GEOM_HOMOGRAPHY (4-point minimal solver) or CS_GEOM_FUNDAMENTAL (7-point, up to 3 models per sample).
 * - Sampling (counter-based, reproducible on a CPU): draw d of sample s is
 *     x = splitmix64(seed + 0x9E3779B97F4A7C15 * ((s << 8) | d)),   idx = ((x >> 32) * numValid) >> 32   (uint64)
 *   where idx indexes the valid pairs in input order and splitmix64(z) is the output of one splitmix64 step from state z:
 *     z += 0x9E3779B97F4A7C15; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9; z = (z ^ (z >> 27)) * 0x94D049BB133111EB;
 *     return z ^ (z >> 31).
 *   A draw that repeats an earlier index of the same sample is skipped (the next draw is d + 1); a sample that has not
 *   found its 4 / 7 distinct indices after 64 draws is degenerate.
 * - Residuals in pixels; a pair is an inlier when its residual is strictly below thresh:
 *     homography: the transfer error |x2 - pi(H x1)|;
 *     fundamental: the Sampson error, (x2^T F x1)^2 / ((F x1)_0^2 + (F x1)_1^2 + (F^T x2)_0^2 + (F^T x2)_1^2) < thresh^2.
 *   Scoring runs in FP32 on coordinates normalised with per-image centroids and one common scale, against the threshold
 *   scaled by the same factor, so these pixel definitions hold up to FP32 rounding.
 * - The model with the most inliers wins (ties: the lowest slot sample*3 + root, roots in ascending order of the pencil
 *   parameter a of det(a F1 + (1 - a) F2) = 0).  It is refitted once on its inliers (8-point for F, needs 8; DLT for H)
 *   and the refit is kept unless it has fewer inliers.  A degenerate sample: fewer than k distinct draws, three of the
 *   four points collinear in either image (H), or a pivot below 1e-9 in the elimination on normalised coordinates.
 * - model_out: row-major 3x3, pixel coordinates; H scaled to H[2][2] = 1, F to unit Frobenius norm with its
 *   largest-magnitude entry positive.  d_inliers: the inlier pairs {i, j} of that model in input order (int pairs,
 *   device, 8-byte aligned); only the first maxInliers are written.
 * Returns the total inlier count, or CS_E_*.  Fewer than 4 (H) / 7 (F) valid pairs, or no non-degenerate sample: 0 and
 * a zero model.  numPairs == 0 returns 0 and a zero model before any CUDA call (cs_verify_stats keeps the previous
 * call).  CS_E_ARG, before any CUDA call, for n < 0, a NULL set with n > 0, numPairs < 0, NULL pairs with
 * numPairs > 0, model not in {1, 2}, numLoops outside [1, 65536], thresh not finite or <= 0, NULL model_out,
 * maxInliers < 0, NULL inliers with maxInliers > 0, and pair or inlier buffers that are not 8-byte aligned or that
 * overlap each other or a record range.  *ms (may be NULL) gets the event time of the call.
 * One call issues 8 kernel launches and synchronises with the host once, at the end; its scratch lives in the
 * per-device context. */
#define CS_GEOM_HOMOGRAPHY  1
#define CS_GEOM_FUNDAMENTAL 2
int cs_verify_pairs(const void *d_s1, int n1, const void *d_s2, int n2, const int *d_pairs, int numPairs,
                    int model, int numLoops, float thresh, unsigned long long seed,
                    double model_out[9], int *d_inliers, int maxInliers, double *ms);
/* Same with host record arrays, a host pair list and a host inlier buffer. */
int cs_verify_pairs_host(const void *h_s1, int n1, const void *h_s2, int n2, const int *h_pairs, int numPairs,
                         int model, int numLoops, float thresh, unsigned long long seed,
                         double model_out[9], int *h_inliers, int maxInliers, double *ms);
/* The last cs_verify_pairs* call on this thread's device: out[0] = valid pairs, [1] = invalid pairs, [2] =
 * non-degenerate samples, [3] = models scored, [4] = the winning slot (sample*3 + root, -1 if none), [5] = its inlier
 * count, [6] = 1 if the refit was kept, [7] = the final inlier count. */
int cs_verify_stats(long long out[8]);

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
/* The describe stage alone (orientations, secondaries, descriptors) on one level image: d_pts[0..n) are records as
 * the detector leaves them (xpos, ypos, scale in level coordinates, subsampling = 2^k with 0 <= k < 8, capacity
 * maxPts records), described in place by the extractor's kernel; secondaries go to slots n.. while they fit, and none
 * for records with subsampling == finestSubsampling (reference quirk Q1).  Returns the record count by the
 * extractor's rule, max(min(primaries, maxPts), min(slots claimed, maxPts)). */
int cs_describe_points(const float *d_img, int width, int height, int pitch, void *d_pts, int n, int maxPts,
                       float finestSubsampling);
/* Steps 1-4 of cs_verify_pairs (validation, normalisation, minimal solvers, scoring) with the same arguments and checks:
 * h_models[3*numLoops][9] receives every slot's model in pixel coordinates with the output scaling of cs_verify_pairs
 * (NaN-filled when the slot is empty), h_counts[3*numLoops] every slot's inlier count and h_norm the normalisation
 * {c1x, c1y, c2x, c2y, s} (u = s * (x - c)).  Returns the number of valid pairs. */
int cs_verify_models(const void *d_s1, int n1, const void *d_s2, int n2, const int *d_pairs, int numPairs, int model,
                     int numLoops, float thresh, unsigned long long seed, double *h_models, int *h_counts,
                     double h_norm[5]);

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
