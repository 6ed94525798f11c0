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
 * "cap32_limit" (the cap's limit, 1..199; default 32), "texture_group_bytes" (the depth-buffer bytes of one image
 * group of cs_texture_mesh, <= 0: 1 GiB).  Returns 0, or CS_E_ARG for an unknown key. */
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
 * cs_alloc_temp (NULL = internal, cached).  Returns numPts.  CS_E_ARG, before any CUDA call,
 * when level 0 (width x height, doubled by scaleUp) is wider or taller than 8193 px: an extremum's
 * position is kept in 13-bit fields.  The same limit holds for cs_extract_host and every
 * cs_extractor_create_*. */
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

/* Calibrated two-view verification (RANSAC for the essential matrix, 5-point minimal solver) and the relative pose:
 * findEssentialMat + recoverPose on the device.  Validity, the pair format, the sampler (5 distinct draws per
 * sample), the order of d_inliers, synchronisation, scratch and the argument checks are those of cs_verify_pairs.
 * - K1, K2: row-major pinhole intrinsics of image 1 and image 2, skew allowed: all entries finite, K[3] = K[6] = K[7] =
 *   0, K[8] = 1, K[0] > 0, K[4] > 0.  Calibrated coordinates, in double from the float record coordinates:
 *     y^ = (y - K[5]) / K[4],   x^ = (x - K[2] - K[1] * y^) / K[0].
 * - Minimal solver (Nister), FP64 on the calibrated coordinates of the 5 drawn pairs: rows {X x, X y, X, Y x, Y y, Y,
 *   x, y, 1} ((x, y) image 1, (X, Y) image 2), their null space by the elimination of cs_verify_pairs (pivot 1e-9;
 *   N0..N3 for the free columns 5..8).  Basis: modified Gram-Schmidt of N0, N1, N2, N3 in that order (each vector minus
 *   its projections on the earlier unit vectors, then divided by its norm; a zero norm makes the sample degenerate),
 *   giving q0..q3, then X = (q0 - q1 + q2 - q3) / 2, Y = (q0 + q1 - q2 - q3) / 2, Z = (q0 - q1 - q2 + q3) / 2,
 *   W = (q0 + q1 + q2 + q3) / 2, and E = x X + y Y + z Z + W.  The ten cubics det E = 0 and
 *   2 E E^T E - tr(E E^T) E = 0 (entry (i, j) is row 1 + 3i + j) in the 20 monomials x^3 y^3 x^2y xy^2 x^2z x^2 y^2z y^2
 *   xyz xy xz^2 xz x yz^2 yz y z^3 z^2 z 1; Gauss-Jordan with partial pivoting on the first ten columns (the first row
 *   of equal magnitude; a pivot at or below 1e-12 of the largest |entry| makes the sample degenerate).  Rows 4 - z*5,
 *   6 - z*7, 8 - z*9 are [x y 1] times polynomials in z; the determinant of that 3x3 matrix (cofactors along its
 *   first row) has degree 10.  Its leading coefficients at or below 1e-12 of the largest |coefficient| are dropped.
 *   Distinct real roots by a Sturm sequence of the monic polynomial p of degree n: S0 = p, S1 = p' / n,
 *   S(k+1) = -rem(S(k-1), S(k)) divided by the magnitude of its leading coefficient.  The sequence ends at a remainder
 *   whose largest |coefficient| is at or below 1e-14 of its dividend's largest; a remainder's leading coefficients at
 *   or below 1e-14 of its own largest |coefficient| are dropped.  Isolation on (-B, B] with Fujiwara's bound
 *   B = 1 + 2 max_k |a(n-k)|^(1/k) (a the monic coefficients, k = 1..n), by bisection at midpoints, left half first,
 *   halves without a root dropped; an interval is refined as one root when it holds one root, when it is narrower than
 *   1e-10 * max(1, |lo|, |hi|), or when more than 62 other intervals are pending (room for 64).  Refinement: bisection
 *   to a width of 1e-10 * max(1, |lo|, |hi|) (on the sign of the polynomial when it changes sign across the interval,
 *   else on the Sturm count, keeping the left half while it holds a root), then up to 3 Newton steps from the
 *   midpoint, each kept only while it stays inside the interval.  Roots ascending in z.  (x, y, 1) is the cross product
 *   of two rows of the evaluated 3x3 matrix, the pair (0,1), (0,2), (1,2) with the largest |third component| (the first
 *   of equals), divided by that component; a root where it is 0 is skipped.  Slot sample*10 + r holds the r-th
 *   remaining solution; a sample is degenerate when it has fewer than 5 distinct draws or a pivot fails.
 * - Residual: the Sampson error in pixels of F = K2^-T E K1^-1, exactly as cs_verify_pairs with CS_GEOM_FUNDAMENTAL
 *   (FP32 on normalised coordinates, the model Fn = T2^-T F T1^-1 at unit norm), so thresh means the same and the F
 *   of a result can go to cs_match_guided(..., CS_GEOM_FUNDAMENTAL, ...).  Ties: the lowest slot.
 * - Refit, once, with at least 8 inliers of the winning model: the 8-point normal matrix on calibrated coordinates of
 *   both images scaled by lambda = s * (K1[0] K1[4] K2[0] K2[4])^(1/4) (s the normalisation scale; not centred), its
 *   smallest eigenvector E' (Jacobi), E = S E' S with S = diag(lambda, lambda, 1), projected to the essential manifold
 *   (below).  Kept unless it has fewer inliers.
 * - Projection: the eigenvectors of E^T E (Jacobi), descending (the lower index first on ties); v1, v2 those of the
 *   two largest eigenvalues, sigma_i their square roots (> 0, else no projection), u_i = E v_i / sigma_i;
 *   Ep = u1 v1^T + u2 v2^T, U = (u1, u2, u1 x u2), V = (v1, v2, v1 x v2).
 * - Outputs: E_out is the projection of the final E (the refit, or the winner (T2 K2)^T Fn (T1 K1)) at unit Frobenius
 *   norm, its largest-magnitude entry positive.  Pose candidates, in this order: (U W V^T, +u3), (U W V^T, -u3),
 *   (U W^T V^T, +u3), (U W^T V^T, -u3), W = [0 -1 0; 1 0 0; 0 0 1]; each is a rotation (det +1) and a unit
 *   translation with E_out proportional to [t]x R, mapping camera-1 points to camera 2 (X2 = R X1 + t).  A final inlier
 *   is in front of a candidate when the least-squares depths of l2 x^2 = l1 R x^1 + t are both > 0, computed in double
 *   as l1 ~ (a.b)(b.t) - (a.t)(b.b), l2 ~ (a.a)(b.t) - (a.b)(a.t) with a = R x^1, b = x^2, and its rays are not parallel:
 *   (a.a)(b.b) - (a.b)^2 > 1e-12 (a.a)(b.b).  R_out, t_out: the candidate with the most inliers in front (the first
 *   of equals).  A planar scene admits two physically valid poses; the one returned is then one of them.
 * Returns the total inlier count, or CS_E_*.  Fewer than 5 valid pairs or no non-degenerate sample: 0 and zero E, R,
 * t.  numPairs == 0 returns 0 and zero E, R, t before any CUDA call.  A final E that cannot be projected leaves E, R, t
 * zero.  CS_E_ARG, before any CUDA call, as cs_verify_pairs (model aside), and for NULL or invalid K1 or K2 and NULL
 * E_out, R_out or t_out.  One call issues 8 kernel launches (flags, compact, norm, 5-point hypotheses, score, arg-max,
 * E refit with the pose, write) and synchronises once, at the end.  The hypothesis kernel uses an 8 KB stack per thread:
 * the first call of a process makes the CUDA driver reserve local memory for every thread that can be resident (about
 * 1.8 GB measured on an H100), which it keeps for the life of the context. */
int cs_verify_essential(const void *d_s1, int n1, const void *d_s2, int n2, const int *d_pairs, int numPairs,
                        const double K1[9], const double K2[9], int numLoops, float thresh, unsigned long long seed,
                        double E_out[9], double R_out[9], double t_out[3], int *d_inliers, int maxInliers, double *ms);
/* Same with host record arrays, a host pair list and a host inlier buffer. */
int cs_verify_essential_host(const void *h_s1, int n1, const void *h_s2, int n2, const int *h_pairs, int numPairs,
                             const double K1[9], const double K2[9], int numLoops, float thresh,
                             unsigned long long seed, double E_out[9], double R_out[9], double t_out[3],
                             int *h_inliers, int maxInliers, double *ms);
/* The last cs_verify_essential* call on this thread's device: [0..7] as cs_verify_stats (the winning slot is
 * sample*10 + root), [8] = the final inliers in front of the chosen pose, [9] = the runner-up candidate's count.
 * cs_verify_stats keeps describing cs_verify_pairs* calls. */
int cs_verify_essential_stats(long long out[10]);

/* Batched verification: J independent jobs in one call, for example every matched pair of an image collection.  A job
 * is one image pair's record sets, pair list and seed; model, numLoops and thresh are common to all jobs. */
typedef struct cs_verify_job {
  const void *s1; int n1;          /* device SiftPoint records, as cs_verify_pairs */
  const void *s2; int n2;
  const int *pairs; int numPairs;  /* device int pairs {i, j}, 8-byte aligned */
  unsigned long long seed;
  int *inliers; int maxInliers;    /* device, 8-byte aligned; NULL allowed when maxInliers == 0 */
} cs_verify_job;
/* - Equivalence: for job p, models_out[p] (E_out[p], R_out[p], t_out[p]), counts_out[p], the first maxInliers inlier
 *   pairs and stats_out[p] equal, bit for bit, what a call on that job's fields alone returns:
 *   cs_verify_pairs(s1, n1, s2, n2, pairs, numPairs, model, numLoops, thresh, seed, ...) and then cs_verify_stats for
 *   cs_verify_pairs_batch; cs_verify_essential with K1s[p], K2s[p] and then cs_verify_essential_stats for
 *   cs_verify_essential_batch.  Every other rule is the single call's: validity, sampler, residuals, ties, refit,
 *   projection, pose and inlier order.  Jobs do not interact: permuting the jobs permutes the results.
 * - Empty jobs: a job with numPairs == 0 gets a zero model (zero E, R and t), count 0 and zero statistics, and launches
 *   nothing.  numJobs == 0 returns 0 before any CUDA call (the outputs may then be NULL).
 * - CS_E_ARG, before any CUDA call, with the first offending job index (jobs[p]) in cs_last_error(): every per-job rule
 *   of cs_verify_pairs / cs_verify_essential (its sets, pair and inlier buffers; model, numLoops and thresh), numJobs
 *   outside [0, 65536], NULL jobs with numJobs > 0, NULL models_out / E_out / R_out / t_out or counts_out, NULL or
 *   invalid K1s / K2s, a total of numPairs over all jobs above INT_MAX, and an inlier buffer that overlaps another
 *   job's inlier buffer, pair list or record range.  Record sets and pair lists are only read, so jobs may share them
 *   (one image's records in many pairs, a set paired with itself).  The overlap test sorts the ranges: O(J log J).
 * - Launches: the non-empty jobs, in order, run in waves.  A wave is the longest run of consecutive non-empty jobs
 *   (empty jobs skipped) whose model-slot scratch, slots per sample x numLoops x 76 bytes per job (3 slots per sample
 *   for F and H, 10 for E), fits 256 MiB; it holds at least one job.  Each wave issues the 8 launches of a single
 *   call, so a batch issues 8 x waves launches (cs_launch_count) with waves = ceil(non-empty jobs / max(1,
 *   floor(256 MiB / (slots per sample x numLoops x 76 B)))).  The call synchronises with the host once, at the end;
 *   its scratch lives in the per-device context.  *ms (may be NULL) gets the event time of the call.
 * - cs_verify_stats and cs_verify_essential_stats keep describing single calls; batch statistics come back only
 *   through stats_out (NULL: not written).
 * models_out[J][9], counts_out[J]; stats_out[J][8] may be NULL.  Returns 0 or CS_E_*. */
int cs_verify_pairs_batch(const cs_verify_job *jobs, int numJobs, int model, int numLoops, float thresh,
                          double *models_out, int *counts_out, long long *stats_out, double *ms);
/* K1s, K2s: [J][9] intrinsics per job; E_out[J][9], R_out[J][9], t_out[J][3], counts_out[J];
 * stats_out[J][10] may be NULL. */
int cs_verify_essential_batch(const cs_verify_job *jobs, int numJobs, const double *K1s, const double *K2s,
                              int numLoops, float thresh, double *E_out, double *R_out, double *t_out,
                              int *counts_out, long long *stats_out, double *ms);

/* Batched ratio matching: J independent jobs of cs_match_ratio in one call, for example every image pair of a
 * collection.  A set is one image's records; a job names two sets and its own pair buffer.  maxRatio, maxDistance and
 * crossCheck are common to all jobs. */
typedef struct cs_match_set {
  const void *pts; int n;          /* device SiftPoint records, only read */
} cs_match_set;
typedef struct cs_match_job {
  int set1, set2;                  /* indices into sets */
  int *pairs; int maxPairs;        /* device int pairs {i, j}, 8-byte aligned; NULL allowed when maxPairs == 0 */
} cs_match_job;
/* - Equivalence: for job p with A = sets[set1] and B = sets[set2], counts_out[p] and the first min(count, maxPairs)
 *   pairs equal, bit for bit, what cs_match_ratio(A.pts, A.n, B.pts, B.n, maxRatio, maxDistance, crossCheck, pairs,
 *   maxPairs, mode, ...) returns and writes, in every mode.  stats_out[p][0..2] equal cs_match_stats()[0..2] after that
 *   call in mode 2 (the groups re-scored, the exact chains and the fallback rows, both directions summed with
 *   crossCheck; the all-exact marker {0, 0, 2^64 - 1} when a value of A or B is not finite or |x| >= 8), and
 *   stats_out[p][3] = 2.  Every job runs the tensor path at any size; the exact kernels serve the rows it cannot
 *   certify.  Jobs do not interact: permuting the jobs permutes the results, and two calls give the same bytes.
 * - Sets are shared: any number of jobs may name a set, in either role, a set may be paired with itself and sets may
 *   overlap each other.  A job with an empty set gets count 0 and zero statistics, and launches nothing.  numJobs == 0,
 *   or only empty jobs, returns 0 before any CUDA call.
 * - CS_E_ARG, before any CUDA call, naming the first offending jobs[p] or sets[s] in cs_last_error(): numSets or
 *   numJobs outside [0, 65536], NULL sets or jobs with a positive count, NULL counts_out with numJobs > 0, a set with
 *   n < 0 or a NULL pts with n > 0, set1 or set2 outside [0, numSets), maxPairs < 0, NULL pairs with maxPairs > 0, a
 *   pair buffer that is not 8-byte aligned, a NaN maxRatio or maxDistance, and a pair buffer that overlaps another
 *   job's pair buffer or any set's records (one sweep over sorted ranges, O((J + S) log(J + S))).
 * - Waves: the non-empty jobs, in order, run in waves.  A wave is the longest run of consecutive non-empty jobs whose
 *   scratch fits 256 MiB; it holds at least one job.  The scratch of a wave counts, once per distinct set it uses,
 *   516 bytes per row of the set rounded up to a multiple of 128 rows (split-FP16 operand tiles and norms; a set is
 *   converted once per wave whatever the number of its jobs), and per direction (one per job, two with crossCheck: the
 *   rows of set 1 against set 2 and the rows of set 2 against set 1) 160 bytes per row of its first set rounded up to
 *   128 rows (top-3 tables) plus 24 bytes per row (neighbour lists, fallback entries).  A call also reserves 20 KiB of
 *   tables per SM and a few words per row for the pair scratch.
 * - Launches: each wave issues 6 kernel launches, whatever its number of jobs and crossCheck (convert, GEMM, resolve,
 *   exact fallback, ratio test, pair writes), so a batch issues 6 x waves (cs_launch_count).  The call synchronises
 *   with the host once, at the end; its scratch lives in the per-device context.  *ms (may be NULL) gets the event
 *   time of the call.  cs_match_stats keeps describing single calls.
 * counts_out[J]; stats_out[J][4] may be NULL.  Returns 0 or CS_E_*. */
int cs_match_ratio_batch(const cs_match_set *sets, int numSets, const cs_match_job *jobs, int numJobs, float maxRatio,
                         float maxDistance, int crossCheck, int *counts_out, unsigned long long *stats_out, double *ms);

/* Guided matching (COLMAP's guided_matching): the two nearest neighbours and the ratio test restricted to the pairs a
 * model admits.  cs_match_knn2_guided has the semantics of cs_match_knn2 (the reference's score, only scores > 0, the
 * order score descending then index ascending, a missing neighbour is (-1, 0.0f)), except that row i of set 1 only
 * considers the j with admissible(i, j).  cs_match_guided is cs_match_ratio on those lists (same rule, cross-check
 * and pair order) and returns the pair count; with crossCheck, row j of set 2 considers the i with admissible(i, j),
 * the same function of (i, j) evaluated on the same operands in the same order.
 * - model: CS_GEOM_HOMOGRAPHY or CS_GEOM_FUNDAMENTAL; model_in: row-major 3x3 mapping set-1 pixels to set-2 pixels (what
 *   cs_verify_pairs writes).  It is scaled to unit Frobenius norm in double (the sum of squares in index order) and
 *   each entry rounded to float, f0..f8; t2 = fl(thresh * thresh).
 * - The predicate, every operation one IEEE FP32 rounding in the stated order, no contraction; (x, y) = set-1 xpos,
 *   ypos and (u, v) = set-2 xpos, ypos:
 *     F: l0 = (f0*x + f1*y) + f2, l1 = (f3*x + f4*y) + f5, l2 = (f6*x + f7*y) + f8, a = l0*l0 + l1*l1;
 *        m0 = (f0*u + f3*v) + f6, m1 = (f1*u + f4*v) + f7, b = m0*m0 + m1*m1; num = (l0*u + l1*v) + l2;
 *        admissible iff num*num < t2 * (a + b)  (the Sampson error below thresh).
 *     H: px = (f0*x + f1*y) + f2, py = (f3*x + f4*y) + f5, pw = (f6*x + f7*y) + f8; dx = u*pw - px, dy = v*pw - py;
 *        admissible iff dx*dx + dy*dy < t2 * (pw*pw)  (the forward transfer error below thresh; pw == 0 admits
 *        nothing).
 *   A record with a non-finite xpos or ypos is admissible with nothing.  cs_verify_pairs scores on normalised
 *   coordinates, so a pair within about 1e-4 px of thresh can be an inlier there and not admissible here.
 * - CS_E_ARG, before any CUDA call: the argument rules of cs_match_knn2 / cs_match_ratio except mode (there is one
 *   path), a model outside {1, 2}, a NULL model_in, a non-finite or all-zero model_in (or one whose norm is not
 *   finite), and thresh not finite or <= 0.  n1 == 0 or n2 == 0 returns 0 and writes nothing.  The records are only
 *   read.  A cs_match_guided call issues 7 kernel launches with or without crossCheck (prep, histogram, scan, scatter,
 *   knn over every direction, ratio test, pair writes), a cs_match_knn2_guided call 5 (no ratio test or pair writes)
 *   (cs_launch_count).  The call synchronises once, at the end; the lists of cs_match_guided live in per-device
 *   scratch. */
int cs_match_knn2_guided(const void *d_s1, int n1, const void *d_s2, int n2, int model, const double model_in[9],
                         float thresh, int *d_idx, float *d_score, double *ms);
int cs_match_guided(const void *d_s1, int n1, const void *d_s2, int n2, int model, const double model_in[9],
                    float thresh, float maxRatio, float maxDistance, int crossCheck, int *d_pairs, int maxPairs,
                    double *ms);
/* Same with host record arrays and a host pairs buffer. */
int cs_match_guided_host(const void *h_s1, int n1, const void *h_s2, int n2, int model, const double model_in[9],
                         float thresh, float maxRatio, float maxDistance, int crossCheck, int *h_pairs, int maxPairs,
                         double *ms);
/* the last guided call on this thread's device: [0] predicate evaluations, [1] admissible pairs (= exact chains run),
 * [2] rows of set 1 with at least one admissible candidate, [3] the same for set 2 in a cross-checked call, else 0 */
int cs_match_guided_stats(unsigned long long out[4]);

/* Batched guided matching: J independent jobs of cs_match_guided in one call, for example every verified image pair of
 * a collection.  Sets and jobs are those of cs_match_ratio_batch; each job has its own model.  thresh, maxRatio,
 * maxDistance and crossCheck are common to all jobs.
 * - models[p]: CS_GEOM_HOMOGRAPHY or CS_GEOM_FUNDAMENTAL; models_in[p]: row-major 3x3 mapping set-1 pixels to set-2
 *   pixels, laid out as cs_verify_pairs_batch's models_out, so that output can be passed in unchanged (for a calibrated
 *   pair, the F of its essential matrix).
 * - Equivalence: for job p with A = sets[set1] and B = sets[set2], counts_out[p] and the first min(count, maxPairs)
 *   pairs equal, bit for bit, what cs_match_guided(A.pts, A.n, B.pts, B.n, models[p], models_in + 9 p, thresh,
 *   maxRatio, maxDistance, crossCheck, pairs, maxPairs, ...) returns and writes, and stats_out[p] equals
 *   cs_match_guided_stats() after that call.  Jobs do not interact: permuting the jobs permutes the results, and two
 *   calls give the same bytes.
 * - Sets are shared: any number of jobs may name a set, in either role, a set may be paired with itself and sets may
 *   overlap each other.  A job with an empty set gets count 0 and zero statistics, and launches nothing.  numJobs == 0,
 *   or only empty jobs, returns 0 before any CUDA call.
 * - CS_E_ARG, before any CUDA call, naming the first offending jobs[p] or sets[s] in cs_last_error(): every rule of
 *   cs_match_ratio_batch, NULL models or models_in with numJobs > 0, and per job every model rule of cs_match_guided
 *   (a model outside {1, 2}, a non-finite or all-zero models_in[p] or one whose norm is not finite, thresh not finite
 *   or <= 0).  A zero model is an error: leave out the jobs whose verification failed.
 * - Waves: the non-empty jobs, in order, run in waves.  A wave is the longest run of consecutive non-empty jobs whose
 *   scratch fits 256 MiB; it holds at least one job.  With c = crossCheck, m = c ? n1 : 1, cap0 = 2 n2 + 64 and
 *   cap1 = c ? 2 n1 + 64 : 1, the scratch of a job of n1 x n2 rows is 256 bytes (header and pair total) plus these
 *   pieces, each rounded up to a multiple of 256 bytes: 4 cap0 and 4 cap1 (cell counts), 32 (n1 + n2) (points),
 *   8 (n1 + n2) (cells), 4 (cap0 + 1) twice and 4 (cap1 + 1) twice (cell starts), 16 n2, 4 n2, 16 n2, 4 n2, 16 m,
 *   4 m, 16 m and 4 m (sorted candidate copies), 8 n1 twice and with c 8 n2 twice (knn lists), 4 ceil(n1 / 32) and
 *   4 ceil(n1 / 1024) (pair scratch).
 * - Launches: each wave issues 7 kernel launches, whatever its number of jobs and crossCheck (prep, histogram, scan,
 *   scatter, knn over every direction of every job, ratio test, pair writes), so a batch issues 7 x waves
 *   (cs_launch_count).  The call synchronises with the host once, at the end; its scratch lives in the per-device
 *   context.  *ms (may be NULL) gets the event time of the call.  cs_match_guided_stats keeps describing single calls.
 * models[J], models_in[J][9], counts_out[J]; stats_out[J][4] may be NULL.  Returns 0 or CS_E_*. */
int cs_match_guided_batch(const cs_match_set *sets, int numSets, const cs_match_job *jobs, int numJobs,
                          const int *models, const double *models_in, float thresh, float maxRatio, float maxDistance,
                          int crossCheck, int *counts_out, unsigned long long *stats_out, double *ms);

/* Feature tracks: the connected components of the features that the pair lists of many image pairs join, for example
 * every job of cs_match_guided_batch or cs_match_ratio_batch, in one call (COLMAP's correspondence graph and track
 * building; OpenMVG's tracks builder).  A list uses the pair convention of cs_match_job, so a batch job's buffer can be
 * passed unchanged with numPairs = min(counts_out[p], maxPairs). */
typedef struct cs_track_list {
  int image1, image2;              /* indices into imageSizes */
  const int *pairs; int numPairs;  /* device int pairs {i, j}, 8-byte aligned: feature i of image1 <-> feature j of image2 */
} cs_track_list;
/* - Features: feature f of image a is valid when 0 <= f < imageSizes[a]; its global id is g = imageSizes[0] + ... +
 *   imageSizes[a - 1] + f, and N is the sum of all sizes.
 * - Pairs: pair {i, j} of lists[p] is valid when i is a valid feature of image1 and j a valid feature of image2; it
 *   joins (image1, i) and (image2, j).  An invalid pair is ignored and counted.  image1 == image2, repeated lists and
 *   repeated pairs are allowed.
 * - Components: a feature is matched when it is an endpoint of at least one valid pair; the components are the
 *   connected components of the matched features.  A component conflicts when it holds two distinct features of the
 *   same image.  It is a track when it has at least minLength features (minLength >= 2) and does not conflict, or
 *   dropConflicting == 0.
 * - Order, defined by value: tracks in ascending order of their smallest global id; the members of a track in
 *   ascending global id, which is ascending (image, feature).  d_members receives int pairs {image, feature},
 *   d_offsets[k] is the number of members before track k, d_trackOf[g] is the track index of feature g or -1.  The
 *   output depends only on the set of valid pairs: permuting the lists, permuting the pairs of a list, swapping a
 *   list's two images together with its pair columns, or adding duplicates leave every byte unchanged, and two calls
 *   give the same bytes.
 * - Returns the track count T, or CS_E_*.  With M the total member count: d_offsets (room for maxTracks + 1 ints, 4-byte
 *   aligned) receives its first min(T, maxTracks) + 1 entries; it may be NULL when maxTracks == 0, and then nothing is
 *   written to it.  d_members (room for maxMembers int pairs, 8-byte aligned) receives the first min(M, maxMembers)
 *   members.  d_trackOf (N ints, 4-byte aligned) may be NULL; otherwise all N entries are written, track indices
 *   >= maxTracks included.
 * - stats_out (may be NULL): [0] valid pairs, [1] invalid pairs, [2] matched features, [3] components, [4] components
 *   of at least minLength features that conflict (whatever dropConflicting is), [5] components below minLength, [6] T,
 *   [7] M.
 * - CS_E_ARG, before any CUDA call, naming the first offending lists[p] or imageSizes[a] in cs_last_error(): numImages
 *   or numLists outside [0, 2^24], NULL imageSizes or lists with a positive count, imageSizes[a] < 0, N above INT_MAX
 *   (named at the image where the sum passes it), image1 or image2 outside [0, numImages), numPairs < 0, NULL pairs
 *   with numPairs > 0, pairs not 8-byte aligned, the total of numPairs above INT_MAX, minLength < 2, maxTracks < 0,
 *   maxMembers < 0, NULL d_offsets with maxTracks > 0, NULL d_members with maxMembers > 0, misaligned output buffers,
 *   and output buffers that overlap each other or any pair list (one sweep over sorted ranges, O(L log L)).  Pair lists
 *   are only read and may overlap each other.
 * - No pairs at all (numLists == 0, or every numPairs 0): returns 0 with zero statistics; d_trackOf (when not NULL) is
 *   filled with -1 and d_offsets[0] (when not NULL) set to 0 by memsets, with no kernel launch; with N == 0 or
 *   d_trackOf NULL, and d_offsets NULL, the call makes no CUDA call.  Lists with pairs but no valid pair: returns 0,
 *   d_trackOf all -1, statistics [1] set.
 * - Launches: a call with pairs issues 8 kernel launches (cs_launch_count), whatever numLists and the pair counts:
 *   init, hook (every pair of every list), compress, run bounds, tile reduce, tile scan, track heads, members.  Between
 *   compress and run bounds, cub::DeviceRadixSort sorts the N (label, global id) pairs over ceil(log2 N) key bits; its
 *   launches (a few, by CUB's own plan) are not counted.  The call synchronises with the host once, at the end; *ms
 *   (may be NULL) gets its event time.
 * - Scratch, in the per-device context: 26 bytes per feature (the sort's four buffers, track index and first member
 *   per label, two flag bytes), 8 bytes per 2048 features, 4 bytes per image, 32 bytes per list with pairs, and the
 *   sort's temporary storage; there is no term per pair or per matched feature.  The pair lists are read in place.
 * imageSizes[numImages], lists[numLists] on the host. */
int cs_build_tracks(const int *imageSizes, int numImages, const cs_track_list *lists, int numLists, int minLength,
                    int dropConflicting, int *d_trackOf, int *d_offsets, int maxTracks, int *d_members, int maxMembers,
                    long long stats_out[8], double *ms);

/* Image retrieval: a visual vocabulary (Sivic & Zisserman 2003; spherical k-means, Dhillon & Modha 2001), the word of
 * every feature, and each image's top-k neighbours by tf-idf as the pair list to match (COLMAP's vocabulary-tree
 * matching, without the tree).
 * - Vocabulary: a device array of numWords SiftPoint records whose data[128] holds the words; every other field is 0.
 *   It is a cs_match_set {d_vocab, numWords}: it can go wherever records go and be saved with the memcpy calls.
 * - Word of a descriptor x: j1 of cs_match_knn2(x, vocab), the lowest index with the largest positive reference score
 *   (the sequential FMA chain), or -1 when no score is positive (an all-zero descriptor).  This is the contract.
 *
 * cs_vocab_assign: d_wordOf[base_a + i] = the word of row i of sets[a], base_a = n_0 + ... + n_{a-1} (the global
 * feature id of cs_build_tracks, so d_wordOf lines up with d_trackOf).
 * - Equivalence: bit for bit cs_match_knn2(sets[a], vocab)'s j1 for every set, in every mode, rows of the exact
 *   fallback and sets caught by the bad-input gate (a value of the set or the vocabulary not finite or |x| >= 8)
 *   included.
 * - Waves: those of cs_match_ratio_batch with crossCheck 0 over the jobs (a, vocabulary), a = 0 .. numSets - 1 (the
 *   vocabulary is one set converted once per wave).  Each wave issues 5 kernel launches (convert, GEMM, resolve, exact
 *   fallback, word copy), so a call issues 5 x waves (cs_launch_count).
 * - stats_out (may be NULL) [5]: the totals over the sets of cs_match_stats' [0] groups re-scored, [1] exact chains and
 *   [2] fallback rows (every row of a gated set), [3] the sets caught by the gate, [4] the waves.
 * - CS_E_ARG, before any CUDA call, naming the offending sets[s] or buffer: numSets outside [0, 65536], NULL sets with
 *   numSets > 0, a set with n < 0 or a NULL pts with n > 0, a feature total above INT_MAX, numWords outside [1, 2^18],
 *   NULL or not 16-byte aligned d_vocab, NULL d_wordOf with features, d_wordOf not 4-byte aligned, and d_wordOf
 *   overlapping the vocabulary or any set's records.  A call without features returns 0 and makes no CUDA call.  The
 *   call synchronises once, at the end; *ms (may be NULL) gets its event time.  Returns 0 or CS_E_*. */
int cs_vocab_assign(const cs_match_set *sets, int numSets, const void *d_vocab, int numWords, int *d_wordOf,
                    unsigned long long stats_out[5], double *ms);

/* cs_vocab_train: Lloyd iterations of spherical k-means over every feature of the sets, M descriptors in global order;
 * writes numWords records to d_vocab.
 * - Start: word k is the descriptor of the k-th distinct index of the draws idx = ((splitmix64(seed +
 *   0x9E3779B97F4A7C15 * counter) >> 32) * M) >> 32, counter = 0, 1, 2, ... (uint64; splitmix64 as cs_verify_pairs),
 *   a repeated index skipped.  Identical start descriptors are allowed: the tie rule empties all but the lowest copy.
 * - Iteration t: (1) every descriptor's word by cs_vocab_assign; (2) the assignments that changed since iteration
 *   t - 1 are counted (all of them at t = 0), and none stops the loop; (3) otherwise, per word with members: s =
 *   the members' descriptors summed per component in float64 in ascending global id, norm = the 128 squares summed in
 *   float64 in ascending component (no fused multiply-add), word = float32(s / sqrt(norm)).  A word without members, or
 *   with norm 0, keeps its descriptor.  maxIterations = 0 returns the start words.
 * - trace_out (may be NULL) [maxIterations][4], float64, per iteration run: the changed assignments, the words without
 *   members (at a stop: those of the previous iteration, whose assignment it repeats), the fallback rows of the
 *   assignment, and the mean best score over the assigned descriptors: per tile of 1024 features thread t (of 256) sums
 *   the scores of tile + 4t .. 4t + 3 in order from 0, then x[t] += x[t + s] for s = 128, 64, .., 1, then the tiles in
 *   ascending order, divided by the assigned count (0 without one).  Rows past the last iteration are 0.
 * - stats_out (may be NULL) [4]: iterations run, 1 if the loop stopped on no change, M, kernel launches.
 * - Launches: 1 (start words), then per iteration the 5 x waves of the assignment and 1 compare, and unless it stops 2
 *   more (run bounds, word update); a stable cub::DeviceRadixSort of (word + 1, global id) pairs between them is not
 *   counted.  The call synchronises with the host once per iteration.  Two calls with the same inputs give the same
 *   bytes.
 * - CS_E_ARG, before any CUDA call: the set checks of cs_vocab_assign, numWords outside [1, 2^18] or above M,
 *   maxIterations outside [0, 1000], NULL or not 16-byte aligned d_vocab, and d_vocab overlapping any set's records.
 * Returns the iterations run, or CS_E_*. */
int cs_vocab_train(const cs_match_set *sets, int numSets, int numWords, int maxIterations, unsigned long long seed,
                   void *d_vocab, double *trace_out, long long stats_out[4], double *ms);

/* cs_retrieve_pairs: every image's top-k neighbours by tf-idf and the deduplicated pair table.  imageSizes (host) and
 * d_wordOf (device, N = the sum of the sizes, in the global order of cs_vocab_assign) give each feature's image and
 * word.
 * - Counts: tf_a(w) = the features of image a with word w; words outside [0, numWords) are ignored.  df_w = the images
 *   with tf > 0; N' = the images with at least one word.
 * - Weights: idf_w = log(N' / df_w) in float64 on the device (0 for df_w = 0), written to d_idf (may be NULL);
 *   x = tf idf, v_a(w) = x / sqrt(sum of x^2 over the image's words in ascending w, float64, no fused multiply-add) (0
 *   when that sum is 0); q_a(w) = rint(v_a(w) 2^22) (round half to even), an int32.
 * - Score: score(a, b) = sum_w q_a(w) q_b(w), exact in int64 (below 2^45 by Cauchy-Schwarz), so the order of the
 *   64-bit atomics that form it reaches no output.  Similarity = score 2^-44 as a double (exact).
 * - d_neighbours [numImages][topK] int, d_scores [numImages][topK] double: the images b != a with score > 0, by score
 *   descending then b ascending, padded with -1 and 0.
 * - d_pairs: {min(a, b), max(a, b)} of every listed neighbour, deduplicated, in ascending (first, second), int pairs
 *   as cs_match_job's; the first min(count, maxPairs) are written.  Returns the full count, or CS_E_*.
 * - Waves: the queries run in consecutive ranges of max(1, floor(256 MiB / (8 numImages))) images (their int64
 *   accumulators).
 * - stats_out (may be NULL) [7]: [0] N', [1] postings (distinct (image, word)), [2] sum of df_w^2, [3] score updates
 *   (sum over w of the squared count of postings with q != 0: those with q = 0 add nothing and are skipped), [4] waves,
 *   [5] the full pair count, [6] ignored features.
 * - Launches: 6 + 2 x waves (keys, postings, idf, weights, word bounds; per wave scatter and top-k select; pair
 *   writes).  cub sorts, run-length encoding and unique passes between them are not counted.  The call synchronises
 *   once, at the end; *ms (may be NULL) gets its event time.
 * - CS_E_ARG, before any CUDA call, naming the offending imageSizes[a] or buffer: numImages outside [0, 65536], NULL
 *   imageSizes with numImages > 0, imageSizes[a] < 0, N above INT_MAX, numWords outside [1, 2^18], topK outside
 *   [1, 1024], maxPairs < 0, NULL d_wordOf with N > 0, NULL d_neighbours or d_scores with numImages > 0, NULL d_pairs
 *   with maxPairs > 0, misaligned buffers (d_wordOf, d_neighbours 4 bytes; d_scores, d_idf, d_pairs 8), and an output
 *   overlapping another output or d_wordOf.  N == 0 returns 0 with zero statistics, writes nothing and makes no CUDA
 *   call. */
int cs_retrieve_pairs(const int *imageSizes, int numImages, const int *d_wordOf, int numWords, int topK,
                      int *d_neighbours, double *d_scores, double *d_idf, int *d_pairs, int maxPairs,
                      long long stats_out[7], double *ms);

/* Triangulation of feature tracks with known cameras (COLMAP's point_triangulator, without bundle adjustment): per
 * track, RANSAC over two-view DLT points, the inliers by reprojection error, one multi-view DLT refit.  The tracks of
 * cs_build_tracks can be passed unchanged: d_offsets, d_members and numMembers = its stats_out[7].
 * - Images and cameras: sets[a] holds image a's records (the indexing of cs_build_tracks' imageSizes).  Camera a maps
 *   a world point X to Xc = R_a X + t_a (the convention of cs_verify_essential's pose); its centre is C_a = -R_a^T t_a.
 *   K_a follows cs_verify_essential's rule, and the calibrated coordinates of a record are its formula, in double from
 *   the float xpos, ypos: y^ = (y - K[5]) / K[4], x^ = (x - K[2] - K[1] * y^) / K[0].  Ks, Rs, ts: row-major
 *   [numImages][9], [numImages][9], [numImages][3] on the host.
 * - Tracks: track k's members are d_members[offsets[k] .. offsets[k+1]) (int pairs {image, feature}).  A track is
 *   malformed when offsets[k] < 0, offsets[k+1] < offsets[k] or offsets[k+1] > numMembers (checked on the device): it
 *   gets no point, is counted, and nothing of its members is read or written.  A member {a, f} is valid when
 *   0 <= a < numImages, 0 <= f < sets[a].n and its xpos and ypos are finite.  V is the number of valid members of a
 *   track; ranks 0 .. V-1 index them in member order.
 * - Hypotheses: when V (V - 1) / 2 <= numTrials, every pair of ranks p < q, in lexicographic order, h = 0, 1, ...;
 *   otherwise numTrials samples h = s = 0 .. numTrials-1, drawn with x = splitmix64(seed + 0x9E3779B97F4A7C15 *
 *   ((k << 24) | (s << 4) | d)) and rank = ((x >> 32) * V) >> 32 for d = 0, 1, ... (64-bit unsigned arithmetic,
 *   splitmix64 as in cs_verify_pairs): p is the first draw and q the next draw different from it; a sample without
 *   two distinct ranks after 16 draws is degenerate and is not evaluated.  V < 2: no hypothesis.
 * - Hypothesis h is the two-view DLT in calibrated coordinates: the rows x^ P[2] - P[0] and y^ P[2] - P[1] of member
 *   p, then of member q (P = [R | t] of the member's image, P[i] its row i), summed into the 4x4 normal matrix, whose
 *   eigenvector of the smallest eigenvalue (cyclic Jacobi, the lowest index on ties) is dehomogenised.  It is
 *   admissible when the two members are of different images, the eigenvector's w is nonzero and the point X is
 *   finite, its depth (R X + t)_2 is > 0 in both cameras, and, with a = X - C_p, b = X - C_q, a.b <= cosMin *
 *   sqrt((a.a) (b.b)), cosMin = cos(minTriAngle * pi / 180) (the triangulation angle is at least minTriAngle degrees).
 * - Inlier: a valid member whose depth d = (R X + t)_2 is > 0 and whose squared pixel reprojection error is strictly
 *   below maxError^2, evaluated in double as (u0 - x d)^2 + (u1 - y d)^2 < maxError^2 d^2 with (u0, u1, d) = K (R X + t)
 *   and (x, y) the record's position.
 * - Winner: the admissible hypothesis with the most inliers, the lowest h on ties.  When it has at least 2 inliers,
 *   one refit: the normal matrix of the rows of all its inliers (in rank order), solved as above; it is kept unless it
 *   is not finite (w = 0 or X not finite) or has fewer inliers.  No depth or angle test applies to the refit.  A track
 *   has a point when a winner exists and the final point's inlier count is >= 2.
 * - Outputs: d_points[k] = the final point, d_counts[k] = its inlier count; a track without a point (malformed
 *   included) gets NaN, NaN, NaN and 0.  For every member of a well-formed track, when the buffer is given:
 *   d_errors = (float)sqrt(e2), e2 the squared pixel error under the final point, +inf when its depth is <= 0, NaN for
 *   an invalid member or a track without a point; d_inlier = 1 for a final inlier, else 0.
 * - Returns the number of tracks with a point, or CS_E_*.  stats_out (may be NULL): [0] well-formed tracks, [1]
 *   malformed tracks, [2] invalid members, [3] hypotheses evaluated (non-degenerate samples), [4] admissible
 *   hypotheses, [5] tracks with a point, [6] refits kept, [7] the sum of the final inlier counts.
 * - Determinism: the outputs are a function of the arguments; two calls give the same bytes, whatever the device's
 *   scheduling (except for a member that two well-formed tracks share, possible only with decreasing offsets: its
 *   outputs come from either track).  They agree with a float64 statement of these rules to rounding, not bit for bit: the device contracts
 *   products into fused multiply-adds, and the refit's sums run in a fixed per-lane order.
 * - CS_E_ARG, before any CUDA call, naming the offending sets[a], camera a (Ks[a], Rs[a], ts[a]) or buffer in
 *   cs_last_error(): numImages outside [0, 2^24], numTracks < 0, numMembers < 0, NULL sets, Ks, Rs or ts with
 *   numImages > 0, NULL d_offsets or d_points or d_counts with numTracks > 0, NULL d_members with numMembers > 0, a set
 *   with n < 0 or a NULL pts with n > 0, K not valid by cs_verify_essential's rule, R not finite, not orthonormal
 *   (|R R^T - I| above 1e-6 in an entry) or with det R <= 0, t not finite, numTrials outside [1, 2^20], maxError not
 *   finite or <= 0, minTriAngle not finite or outside [0, 180), d_offsets or d_counts or d_errors not 4-byte aligned,
 *   d_members or d_points not 8-byte aligned, and an output (d_points [numTracks][3] doubles, d_counts, d_errors,
 *   d_inlier) that overlaps another output, d_offsets (numTracks + 1 ints), d_members or any set's records (one sweep
 *   over sorted ranges).  numTracks == 0 returns 0 with zero statistics and makes no CUDA call.
 * - Launches: 1 kernel launch (cs_launch_count), whatever numTracks and the track lengths: a warp per track, claimed
 *   from a queue by one resident wave of CTAs.  The call synchronises with the host once, at the end; *ms (may be
 *   NULL) gets its event time.  Scratch, in the per-device context: 256 bytes, 280 bytes per image (the camera table)
 *   and 16 bytes per member (valid members past the 128 a warp stages in shared memory). */
int cs_triangulate_tracks(const cs_match_set *sets, int numImages, const double *Ks, const double *Rs, const double *ts,
                          const int *d_offsets, int numTracks, const int *d_members, int numMembers, int numTrials,
                          double maxError, double minTriAngle, unsigned long long seed, double *d_points, int *d_counts,
                          float *d_errors, unsigned char *d_inlier, long long stats_out[8], double *ms);

/* Camera registration against known 3-D points (COLMAP's image_registrator, OpenCV's solvePnPRansac), many images in
 * one call: per job, RANSAC over Lambda Twist P3P poses (Persson & Nordberg, ECCV 2018) in FP64, the inliers by the
 * reprojection rule of cs_triangulate_tracks, then one Levenberg-Marquardt refinement.  cs_build_tracks' d_trackOf
 * (offset by the image's global base) and cs_triangulate_tracks' d_points go in unchanged, and R, t come out in the
 * convention cs_triangulate_tracks takes. */
typedef struct cs_pose_job {
  const void *pts; int n;          /* device SiftPoint records of the image to register */
  const int *pointOf;              /* device int[n]: the 3-D point of feature f, or < 0 for none */
  unsigned long long seed;
  float *errors;                   /* device float[n] or NULL: pixel error of every feature under the final pose */
  unsigned char *inlier;           /* device byte[n] or NULL: 1 for a final inlier */
} cs_pose_job;
/* - Correspondences: feature f of job p is valid when 0 <= pointOf[f] < numPoints, the three coordinates of that
 *   point are finite and the record's xpos and ypos are finite (so triangulation's NaN rows, "no point", are skipped).
 *   V is the number of valid correspondences; ranks 0 .. V-1 index them in feature order.  Features may share a point.
 *   A feature with pointOf[f] >= 0 that is not valid is counted as invalid.
 * - K (Ks[p], row-major) follows cs_verify_essential's rule.  The bearing of a correspondence is (x^, y^, 1) divided by
 *   sqrt(x^ x^ + y^ y^ + 1), computed in double, with x^, y^ the calibrated coordinates of cs_verify_essential.
 * - Sampler: cs_verify_pairs' rule with 3 distinct draws over the V ranks: draw d of sample s is
 *   ((x >> 32) * V) >> 32 with x = splitmix64(seed + 0x9E3779B97F4A7C15 * ((s << 8) | d)), repeats skipped, at most
 *   64 draws; samples s = 0 .. numLoops-1.  Y_k, X_k (k = 0, 1, 2) are the bearings and world points in draw order.
 * - Minimal solver (FP64): d12 = X0 - X1, d13 = X0 - X2, d23 = X1 - X2, aij = |dij|^2, n = d12 x d13;
 *   cij = Yi . Yj, sij = 1 - cij^2, bij = -2 cij.  The sample is degenerate when |n|^2 <= 1e-10 a12 a13 (collinear
 *   world points) or some sij <= 1e-10 (near-parallel bearings).  With blob = c12 c23 c13 - 1:
 *     p3 = a13 (a23 s13 - a13 s23),
 *     p2 = 2 blob a23 a13 + a13 (2 a12 + a13) s23 + a23 (a23 - a12) s13,
 *     p1 = a23 (a13 - a23) s12 - a12^2 s23 - 2 a12 (blob a23 + a13 s23),
 *     p0 = a12 (a12 s23 - a23 s12);
 *   p3 == 0 is degenerate.  g is the largest real root of g^3 + (p2/p3) g^2 + (p1/p3) g + p0/p3: the closed form
 *   (Cardano when the discriminant q^2/4 + p^3/27 of the depressed cubic is >= 0, else 2 sqrt(-p/3) cos(acos(...)/3)),
 *   then 2 Newton steps, each taken when the derivative is nonzero and the result finite.  D0 = D1 - g D2 is
 *     [a23 (1 - g),  a23 b12 / 2,          -a23 b13 g / 2;
 *      .,            a23 - a12 + a13 g,    b23 (a13 g - a12) / 2;
 *      .,            .,                    g (a13 - a23) - a12]  (symmetric; a non-finite entry is degenerate),
 *   decomposed by the cyclic Jacobi of the verifiers (vp_jacobi<3>, not the closed form with the known zero
 *   eigenvalue).  e0, e1 are its eigenvalues of largest and second largest magnitude (the lower index first on ties),
 *   u0, u1 their eigenvectors; e0 == 0 is degenerate; v = sqrt(max(0, -e1 / e0)).  For s = +v, then s = -v:
 *   w2 = 1 / (s u1[0] - u0[0]), w0 = (u0[1] - s u1[1]) w2, w1 = (u0[2] - s u1[2]) w2 (so l1 = w0 l2 + w1 l3), and the
 *   quadratic tau^2 + B tau + C = 0 with qa = 1 / ((a13 - a12) w1^2 - a12 b13 w1 - a12),
 *   B = (a13 b12 w1 - a12 b13 w0 - 2 w0 w1 (a12 - a13)) qa, C = ((a13 - a12) w0^2 + a13 b12 w0 + a13) qa.  When
 *   B^2 - 4 C >= 0: tau1 = (-B + sqrt) / 2 if B < 0 else (-B - sqrt) / 2, tau2 = C / tau1 (NaN when tau1 == 0); for
 *   tau1, then tau2, when tau > 0 and dd = a23 / (tau (b23 + tau) + 1) > 0: l2 = sqrt(dd), l3 = tau l2,
 *   l1 = w0 l2 + w1 l3, kept when l1 > 0.  Each kept (l1, l2, l3) takes up to 5 Newton steps on the three equations
 *   li^2 + lj^2 + bij li lj = aij (the 3x3 Jacobian inverted by its adjugate; a step is taken only when its
 *   determinant is nonzero and the result is finite and lowers |r12| + |r13| + |r23|, else the steps stop), and is
 *   dropped unless all three are finite and > 0.  Alignment: with Ck = lk Yk, R = [C0 - C1, C0 - C2, (C0 - C1) x
 *   (C0 - C2)] [d12, d13, n]^-1 (the inverse's rows (d13 x n, n x d12, d12 x d13) / (d12 . (d13 x n))),
 *   t = C0 - R X0; a pose with a non-finite entry is dropped.  Slot sample*4 + r holds the r-th remaining pose; a
 *   degenerate sample is one with fewer than 3 distinct draws or one that trips a test above.
 * - Inlier (FP64, exactly cs_triangulate_tracks' test and fma chain): depth d = (R X + t)_2 > 0 and
 *   (u0 - x d)^2 + (u1 - y d)^2 < maxError^2 d^2, (u0, u1, d) = K (R X + t), through P = K [R | t].
 * - Winner: the slot with the most inliers, the lowest slot on ties.
 * - Refinement, once, when the winner has at least 3 inliers: Levenberg-Marquardt on the sum of squared pixel
 *   residuals (K0 a + K1 b + K2 - x, K4 b + K5 - y), (a, b) = (Xc0, Xc1) / Xc2, Xc = R X + t, over the winner's
 *   inliers in rank order.  Update R <- exp([w]x) R, t <- exp([w]x) t + delta (Rodrigues, I + A [w]x + B [w]x^2 with
 *   A = sin th / th, B = 2 sin^2(th / 2) / th^2, A = 1, B = 1/2 at th = 0), so the Jacobian row of a residual with
 *   gradient gr = d(pixel) / d(Xc) is (Xc x gr, gr): gr_x = (K0, K1, -(K0 a + K1 b)) / Xc2, gr_y = (0, K4, -K4 b) / Xc2.
 *   The 28 sums per residual, x then y of each correspondence: H = J^T J (21, upper triangle row by row), g = J^T r
 *   (6), the cost r^T r.  The step solves (H + lambda diag(H)) step = -g by Cholesky (a pivot not > 0 or not finite
 *   rejects the step); lambda starts at 1e-3, x10 on a rejected step, /10 on an accepted one.  A step is accepted when
 *   every residual point stays in front (Xc2 > 0) and the cost decreases.  At most 20 iterations; it stops after an
 *   accepted step whose largest |component| is <= 1e-12 or whose cost decrease is <= 1e-12 of the previous cost.  The
 *   refined pose is kept unless it is not finite or has fewer inliers than the winner.
 * - Outputs: R_out[p] (row-major), t_out[p] with X_c = R X + t; counts_out[p] the final inlier count.  A job without
 *   a pose (V < 3, no pose scored, or a final count < 3) gets zero R and t and count 0.  Per feature, when the buffer
 *   is given: errors[f] = (float)sqrt(e2), e2 the squared pixel error under the final pose, +inf when its depth is
 *   <= 0, NaN for a feature that is not a valid correspondence or in a job without a pose; inlier[f] = 1 for a final
 *   inlier, else 0.  stats_out[p] (may be NULL): [0] valid correspondences, [1] invalid ones, [2] non-degenerate
 *   samples, [3] poses scored, [4] the winning slot (-1 if none), [5] its count, [6] 1 when the refinement was kept,
 *   [7] the final count (counts_out[p]).
 * - Returns the number of jobs with a pose, or CS_E_*.
 * - Batch: jobs do not interact; permuting the jobs permutes the results, a job's results are bit-identical alone or
 *   in any batch, and two calls give the same bytes.  Empty jobs (n == 0) get zero outputs and statistics and launch
 *   nothing; numJobs == 0 returns 0 before any CUDA call.  Sums of the refinement run per lane of a warp and combine
 *   by a fixed butterfly, so they agree with a float64 statement of these rules to rounding, not bit for bit.
 * - CS_E_ARG, before any CUDA call, naming the offending jobs[p] in cs_last_error(): numJobs outside [0, 65536], NULL
 *   jobs or Ks with numJobs > 0, numPoints < 0, NULL d_points with numPoints > 0, d_points not 8-byte aligned, n < 0,
 *   NULL pts or pointOf with n > 0, pointOf or errors not 4-byte aligned, an invalid Ks[p], numLoops outside
 *   [1, 65536], maxError not finite or <= 0, NULL R_out, t_out or counts_out with numJobs > 0, and a per-feature
 *   output that overlaps another output, any record range, any pointOf or d_points (one sweep over sorted ranges).
 * - Waves: the non-empty jobs, in order, run in waves of floor(256 MiB / (4 x numLoops x 100 B)) jobs (clamped to
 *   [1, 65536]; a slot is 12 doubles and a count).  Each wave issues 5 kernel launches (gather, hypotheses, score,
 *   arg-max, refine), so a batch issues 5 x waves (cs_launch_count).  The call synchronises with the host once, at
 *   the end; its scratch lives in the per-device context.  *ms (may be NULL) gets the event time of the call.
 * d_points [numPoints][3]; Ks [J][9]; R_out [J][9], t_out [J][3], counts_out [J]; stats_out [J][8] or NULL. */
int cs_absolute_pose_batch(const double *d_points, int numPoints, const cs_pose_job *jobs, int numJobs,
                           const double *Ks, int numLoops, double maxError, double *R_out, double *t_out,
                           int *counts_out, long long *stats_out, double *ms);

/* Bundle adjustment (Triggs et al. 2000; COLMAP's bundle_adjuster): Levenberg-Marquardt over every camera pose and
 * track point at once, the points eliminated by the Schur complement and the reduced camera system solved by
 * preconditioned conjugate gradients (Agarwal et al., ECCV 2010; Wu et al., CVPR 2011).  It takes what
 * cs_triangulate_tracks takes and returns (sets, Ks, Rs, ts, d_offsets, d_members) and the points it wrote.
 * - Observations: tracks, malformed tracks and valid members follow cs_triangulate_tracks.  A member of a well-formed
 *   track is used when it is valid, d_use is NULL or d_use[m] != 0, the track's point is finite, and the point's depth
 *   (R X + t)_2 is > 0 at the input parameters.  A track whose point has at least 2 used observations takes part;
 *   otherwise its observations are dropped and its point is left unchanged, byte for byte.  Observation o runs over the
 *   used observations of the participating tracks, in track order, then member order.
 * - Cameras: fixed[a] (host bytes; NULL = every image free) is 0 (free: 6 parameters), 1 (held), or 2, 3, 4 (free but
 *   for component fixed[a] - 2 of t, held: COLMAP's scale gauge).  An image with no used observation is held.  K is not
 *   adjusted.  Held images and held components come back bit for bit.
 * - Residual (cs_absolute_pose_batch's): r = (K0 a + K1 b + K2 - x, K4 b + K5 - y), (a, b) = (Xc0, Xc1) / Xc2,
 *   Xc = R X + t.  Update R <- exp([w]x) R (the Rodrigues rule of cs_absolute_pose_batch), t <- t + delta,
 *   X <- X + dX; with gr_x = (K0, K1, -(K0 a + K1 b)) / Xc2, gr_y = (0, K4, -K4 b) / Xc2 the Jacobian rows are
 *   ((R X) x gr, gr) for the camera (w, delta) and gr^T R for the point.  The cost is the sum of r^T r over the used
 *   observations.
 * - LM: H + lambda D, D = diag(H) clamped to [1e-6, 1e32]; lambda starts at 1e-3, /10 after an accepted step, x10
 *   after a rejected one.  A step is accepted when the linear solve succeeded, every used observation stays in front
 *   (Xc2 > 0) and the cost decreases.  The loop stops after maxIterations iterations (accepted or rejected), after an
 *   accepted step with previous cost - new cost <= 1e-10 previous cost, or when lambda exceeds 1e16 after a rejection.
 *   maxIterations = 0, or no used observation, evaluates only.
 * - Linear solve of [U* W; W^T V*] [dc; dp] = -[g_c; g_p] (U, V the camera and point blocks of J^T J, W = J_c^T J_p):
 *   every V*_k by Cholesky, then S dc = b~ with S = U* - W V*^-1 W^T and b~ = -g_c + W V*^-1 g_p, restricted to the
 *   free components (a held component's row and column are the identity's, its b~ entry 0).  Preconditioned CG from
 *   dc = 0: the preconditioner is S's 6 x 6 diagonal block per camera (U*_a - sum over the used observations o of image
 *   a of W_o V*_k^-1 W_ak^T, W_ak the sum of W over track k's observations in image a) by Cholesky; with z = M^-1 r,
 *   p = z + beta p, alpha = r.z / p.S p, beta = r.z(new) / r.z(old).  CG stops before an iteration when
 *   r.r <= linearTol^2 b~.b~ (so with no free camera parameter it runs none: structure only), after
 *   maxLinearIterations iterations, or when p.S p is not > 0.  Then dp_k = V*_k^-1 (-g_k - sum_o J_p^T J_c dc_a).  A
 *   Cholesky pivot that is not > 0 or not finite anywhere rejects the step without evaluating it.
 * - Outputs: R_out [numImages][9], t_out [numImages][3] (may alias Rs, ts exactly); d_points adjusted in place;
 *   for every member of a well-formed track, when the buffer is given, under the final parameters: d_errors and
 *   d_inlier by cs_triangulate_tracks' output rule with maxError (NaN and 0 for an invalid member or a non-finite
 *   point).  cost_out = {initial, final}.  trace_out (may be NULL) [maxIterations][4]: per iteration {the candidate's
 *   cost (NaN when the solve failed), lambda, CG iterations, 1 if accepted}; rows past the last iteration are 0.
 *   stats_out (may be NULL): [0] well-formed tracks, [1] malformed tracks, [2] invalid members, [3] used observations,
 *   [4] points adjusted, [5] free camera parameters, [6] LM iterations, [7] CG iterations in all.
 * - Returns the number of accepted steps, or CS_E_*.
 * - Determinism: every sum has a fixed order that depends on the data only, and no scratch word is rewritten before
 *   every CTA has read it, so two calls give the same bytes whatever the number of images.  Per
 *   point: its observations in order.  Per camera: its observations in order o, cut at multiples of 256 of the
 *   camera-sorted list; a piece is summed by a warp (lane l takes l, l + 32, ..., then an xor butterfly) and the pieces
 *   in ascending order.  Totals over tracks (the cost): tiles of 256 tracks (warp butterflies, then the 8 warps in
 *   order); over cameras (the CG dot products): tiles of 32 cameras (a butterfly); the tile partials lane-strided in
 *   ascending order, then a butterfly.  The results agree with a float64 statement of these rules to rounding.
 * - CS_E_ARG, before any CUDA call, naming the offending sets[a], camera a or buffer in cs_last_error(): every check of
 *   cs_triangulate_tracks but numTrials and minTriAngle (d_counts is not an argument), a fixed[a] outside 0..4,
 *   maxIterations outside [0, 1000], maxLinearIterations outside [1, 10000], linearTol not in (0, 1), NULL R_out or
 *   t_out or cost_out with numImages > 0, and an output (d_points, d_errors, d_inlier) that overlaps another output,
 *   d_offsets, d_members, d_use or any set's records (one sweep over sorted ranges).  numTracks == 0 returns 0
 *   with R_out = Rs, t_out = ts, zero costs, trace and statistics, and makes no CUDA call.  numImages == 0 with
 *   numTracks > 0 runs on the device like any call: every member is invalid, but the tracks (d_offsets) are device
 *   memory, and the well-formed tracks' member outputs (NaN and 0) and the statistics are written from them.
 * - Launches: 3 kernel launches (cs_launch_count) whatever the sizes and iteration counts: the count and fill kernels
 *   and one cooperative kernel (a resident wave, SMs x occupancy CTAs of 256 threads) that runs the whole LM loop with
 *   grid barriers between its phases; a cub scan and sort (not counted) run between them.  The call synchronises with
 *   the host once, at the end; *ms (may be NULL) gets its event time.  Scratch, in the per-device context: 1 392
 *   bytes per image (its state and camera pieces), 176 per track, 200 per member (the observation, J_c, J_p and r,
 *   the sort keys), 432 per 256 members, 36 per LM iteration, plus the cub scan and sort storage; pinned, 944 bytes
 *   per image and 32 per LM iteration. */
int cs_bundle_adjust(const cs_match_set *sets, int numImages, const double *Ks, const double *Rs, const double *ts,
                     const unsigned char *fixed, const int *d_offsets, int numTracks, const int *d_members,
                     int numMembers, const unsigned char *d_use, double *d_points, int maxIterations,
                     int maxLinearIterations, double linearTol, double maxError, double *R_out, double *t_out,
                     float *d_errors, unsigned char *d_inlier, double cost_out[2], double *trace_out,
                     long long stats_out[8], double *ms);

/* Self-calibrating bundle adjustment (COLMAP's RADIAL camera, generalised to the full upper-triangular K): everything
 * cs_bundle_adjust does, with per-image focal length and radial distortion refined and a robust loss.  cs_bundle_adjust
 * is this call with dists = NULL, refine = NULL, loss = 0, K_out = dist_out = NULL.
 * - Camera model, per image: K (K0 = fx, K1 = skew, K2 = cx, K4 = fy, K5 = cy) and k = (k1, k2) = dists[a] (NULL: all
 *   zero).  With Xc = R X + t: (a, b) = (Xc0, Xc1) / Xc2, rho2 = a^2 + b^2, D = 1 + k1 rho2 + k2 rho2^2,
 *   (a', b') = D (a, b), r = (K0 a' + K1 b' + K2 - x, K4 b' + K5 - y).  With k = 0 this is cs_bundle_adjust's residual.
 * - Refined intrinsics: refine[a] (host bytes; NULL = none) has bit 0 the focal f = K0, bit 1 k1, bit 2 k2.  Update
 *   f <- f + df with K1 / K0 and K4 / K0 held (K0c = K0 + df, K1c = K1 (K0c / K0), K4c = K4 (K0c / K0)),
 *   k1 <- k1 + dk1, k2 <- k2 + dk2.  The principal point is not refined.  Intrinsics are held exactly as pose
 *   components are: fixed governs the pose, refine the intrinsics, an image with no used observation holds everything,
 *   and held values come back bit for bit.
 * - Jacobian: with Dp = 2 (k1 + 2 k2 rho2), d(a', b') / d(a, b) = [D + Dp a^2, Dp a b; Dp a b, D + Dp b^2] = Dd and
 *   d(u, v) / d(a, b) = [K0 K1; 0 K4] Dd, the rows gr = d(u, v) / d(Xc) give the pose and point rows as in
 *   cs_bundle_adjust; d(u, v) / df = (K0 a' + K1 b', K4 b') / K0, d(u, v) / dk1 = (K0 a + K1 b, K4 b) rho2, and
 *   d(u, v) / dk2 = that times rho2.
 * - Loss on s = r^T r of each used observation, scale c = lossScale > 0 pixels, applied as c^2 rho(s / c^2):
 *   loss 0 trivial rho(s) = s; 1 soft-L1 rho(s) = 2 (sqrt(1 + s) - 1), computed as 2 s / (sqrt(1 + s) + 1); 2 Cauchy
 *   rho(s) = log(1 + s) (log1p).  The cost is the sum over the used observations (no 1/2).  Linearisation follows
 *   Ceres's corrector: for these losses rho'' <= 0, so it reduces to scaling the observation's r and both Jacobian
 *   blocks by sqrt(rho'(s / c^2)) (1 / sqrt(sqrt(1 + u)) soft-L1, 1 / sqrt(1 + u) Cauchy, u = s / c^2), taken at each
 *   relinearisation; the candidate's cost uses the same rho.
 * - Camera block: NC = 6 (w, delta) when no image refines an intrinsic and every k is 0 (0.0 or -0.0), else NC = 9
 *   (w, delta, f, k1, k2) for every image.  NC = 6 with the trivial loss is cs_bundle_adjust's kernel, byte for byte.
 *   Everything of cs_bundle_adjust that is per camera grows to NC: U, g_c, the Schur term, the preconditioner block and
 *   its Cholesky, CG's vectors.  LM additionally rejects a step after which a refined focal is not > 0.
 * - Outputs as cs_bundle_adjust's, plus K_out [numImages][9] (the final K, row-major, K[6..8] = (0, 0, 1)) and
 *   dist_out [numImages][2] (final k1, k2); either may be NULL, and K_out may equal Ks, dist_out dists, R_out Rs and
 *   t_out ts exactly.  With NC = 6 they are the input's (zeros for NULL dists).  stats_out[5] counts the free
 *   intrinsic parameters too.  Member outputs under the final parameters: with NC = 6 cs_bundle_adjust's rule; with
 *   NC = 9 err = (float)sqrt(r^T r) of the residual above (inf when Xc2 <= 0), inlier when Xc2 > 0 and
 *   r^T r < maxError^2.
 * - Determinism, launches and the fixed summation orders are cs_bundle_adjust's: 3 kernel launches, no floating-point
 *   atomics, two calls give the same bytes.  Scratch with NC = 9: 2 400 bytes per image (1 536 of state, 864 of camera
 *   pieces), 176 per track, 248 per member (the observation, J_c, J_p and r, the sort keys), 864 per 256 members,
 *   36 per LM iteration, plus the cub storage; pinned, 1 536 bytes per image and 32 per LM iteration.
 * - CS_E_ARG, before any CUDA call: every check of cs_bundle_adjust (naming cs_bundle_adjust_intrinsics), a refine[a]
 *   > 7, loss outside 0..2, lossScale not finite or not > 0, a non-finite dists[a], and a host output (K_out, dist_out,
 *   R_out, t_out) that overlaps another output or an input (Ks, dists, Rs, ts) other than exactly its own.
 *   numTracks == 0 returns 0 with the inputs copied to the outputs and makes no CUDA call.
 * dists [numImages][2] or NULL; refine [numImages] or NULL. */
int cs_bundle_adjust_intrinsics(const cs_match_set *sets, int numImages, const double *Ks, const double *dists,
                                const unsigned char *refine, int loss, double lossScale, const double *Rs,
                                const double *ts, const unsigned char *fixed, const int *d_offsets, int numTracks,
                                const int *d_members, int numMembers, const unsigned char *d_use, double *d_points,
                                int maxIterations, int maxLinearIterations, double linearTol, double maxError,
                                double *K_out, double *dist_out, double *R_out, double *t_out, float *d_errors,
                                unsigned char *d_inlier, double cost_out[2], double *trace_out, long long stats_out[8],
                                double *ms);

/* Undistortion of records under cs_bundle_adjust_intrinsics' radial model, so that triangulation and absolute pose
 * (pinhole) can use a refined camera: every record of sets[a] goes to d_out[a] (device, sets[a].n records) with its
 * position corrected under Ks[a] and dists[a] (NULL: all zero) and every other field copied byte for byte.  Orientation
 * and scale are not corrected.
 * - Rule (float64): b = (y - K5) / K4, a = (x - K2 - K1 b) / K0, r_d = sqrt(a^2 + b^2).  Radial distortion keeps the
 *   direction, so r_u solves r_u (1 + k1 r_u^2 + k2 r_u^4) = r_d: Newton's method from r_u = r_d, at most 20
 *   iterations; an iteration with derivative d = 1 + 3 k1 r_u^2 + 5 k2 r_u^4 not > 0 fails, else it takes
 *   r_u -= (r_u (1 + k1 r_u^2 + k2 r_u^4) - r_d) / d and converges when that step's |step| <= 1e-12 r_d.  The output
 *   position is (K0 a s + K1 b s + K2, K4 b s + K5) with s = r_u / r_d (1 when r_d = 0), rounded to float.  A record
 *   gets NaN positions when the solve fails or does not converge, or when d <= 0 at the final r_u; NaN makes it an
 *   invalid member for every track stage.  A non-finite input position gives NaN.
 * - d_out[a] may equal sets[a].pts exactly (in place); otherwise it overlaps no other output and no set's records.
 * - Returns 0 or CS_E_*.  One kernel launch (a thread per record); the call synchronises once, *ms (may be NULL) gets
 *   its event time; no records make no CUDA call.  CS_E_ARG, before any CUDA call, naming the argument: numImages
 *   outside [0, 2^24], NULL sets, Ks or d_out with numImages > 0, a set with records and no pointer, an invalid Ks[a]
 *   (cs_verify_essential's rule), a non-finite dists[a], NULL or not 4-byte aligned d_out[a] for a set with records,
 *   and an overlap (one sweep over sorted ranges). */
int cs_undistort_records(const cs_match_set *sets, int numImages, const double *Ks, const double *dists,
                         void *const *d_out, double *ms);

/* Rotation averaging (Chatterjee and Govindu, ICCV 2013 / TPAMI 2018; the first stage of global structure from
 * motion, as in Theia, OpenMVG and GLOMAP): every image's absolute rotation from the relative rotations of the verified
 * image pairs, in one call.  The inputs are host arrays laid out as cs_verify_essential_batch returns them.
 * - Graph: edge e joins images i = edges[2e] and j = edges[2e + 1] with the relative rotation Q_e = Rrel[e] (row-major,
 *   X_j = Q_e X_i + t, so R_j ~ Q_e R_i) and a weight w0_e = weights[e] > 0 (for example the inlier count).  R maps
 *   world to camera coordinates, as everywhere in this API.
 * - Start (on the host): a maximum spanning tree by weight, Kruskal's algorithm over the edges sorted by weight
 *   descending, ties to the lower edge index.  R_ref = I for refImage; then a breadth-first walk from refImage, each
 *   image's tree edges in ascending edge index, gives an unvisited neighbour R_j = Q_e R_i (from i) or R_i = Q_e^T R_j
 *   (from j).  The images the walk visits are reached; the others get NaN rotations.  An edge is active when its images
 *   are reached (both are, or neither).
 * - Residual of an active edge: D_e = R_j^T Q_e R_i (the discrepancy in the world frame) and rho_e = log D_e, the
 *   rotation vector: c = (tr D - 1) / 2, v the axial vector of (D - D^T) / 2, s = |v|, theta_e = atan2(s, c); for
 *   c > 0 rho = v theta / s (v when s = 0), else rho = theta a, a the unit axis from (D + D^T) / 2 = c I + (1 - c) a a^T
 *   through its largest diagonal entry (the first on ties) and signed so that a.v >= 0.
 * - Loss: sigma = sigmaDeg pi / 180 radians; with sigmaDeg = 0 the squared loss, cost_e = w0_e theta_e^2 and IRLS weight
 *   w_e = w0_e; else Geman-McClure, q = sigma^2 / (theta_e^2 + sigma^2), cost_e = w0_e theta_e^2 q and w_e = w0_e q^2
 *   (rho'(theta) / (2 theta)).  The cost is the sum over the active edges.
 * - Linearisation: a free image's tangent x_i is in the world frame and moves it by R_i <- R_i exp([x_i]x), computed as
 *   the left update exp([R_i x_i]x) R_i (vp_rotate).  Then D_e <- exp(-[x_j]x) D_e exp([x_i]x), and to first order
 *   rho_e(x) = rho_e + Jr^-1(rho_e) x_i - Jl^-1(rho_e) x_j (the right and left Jacobians of SO(3)).  Since
 *   Jr^-T(rho) rho = Jl^-T(rho) rho = rho, the cost's gradient is exactly that of the linear model rho_e + x_i - x_j:
 *   the model has the exact first-order cost, and its Hessian, the weighted graph Laplacian (x) I3, differs from
 *   Gauss-Newton's by O(|rho|).  Each iteration minimises sum_e w_e |rho_e + x_i - x_j|^2 over the free images (reached,
 *   not refImage; x_ref = 0): L x = b with (L x)_a = sum over a's active edges of w_e (x_a - x_other) and
 *   b_a = sum over a's edges of +w_e rho_e (a = j) or -w_e rho_e (a = i).
 * - Solve: Jacobi-preconditioned CG from x = 0, z = r / diag(L), as cs_bundle_adjust's CG (p = z + beta p,
 *   alpha = r.z / p.L p, beta = r.z(new) / r.z(old)); it stops before an iteration when r.r <= linearTol^2 b.b, after
 *   maxLinearIterations iterations, or when p.L p is not > 0.  Every free image then takes its update.
 * - Loop: the iteration above (weights and residuals at the current rotations), at most maxIterations times; it stops
 *   after an iteration whose largest |x_a| is <= 1e-12.  maxIterations = 0 evaluates the start only.
 * - Outputs: R_out [numImages][9] (NaN for an image not reached).  residuals_out [numEdges] (may be NULL): theta_e in
 *   degrees under the final rotations, NaN for an inactive edge; inlier_out [numEdges] (may be NULL): 1 when that angle
 *   is < maxAngleDeg (the filter for positioning and guided matching).  cost_out = {at the start, final}.  trace_out
 *   (may be NULL) [maxIterations][3]: per iteration {the cost at its start, CG iterations, largest |x_a|}; rows past
 *   the last iteration are 0.  stats_out (may be NULL): [0] active edges, [1] tree edges used (images reached - 1),
 *   [2] images reached, [3] iterations, [4] CG iterations in all, [5] inlier edges.  ms_out (may be NULL): {the host's
 *   spanning tree and tables, the device part (event time)} in milliseconds.  Returns the iterations run, or CS_E_*.
 * - Determinism: every sum has a fixed order that depends on the data only and no floating-point atomics are used, so
 *   two calls give the same bytes.  Per image: its incidences (image, 2 e + side) sorted by image (a stable radix sort,
 *   so in edge order), cut at multiples of 256 of that list, a piece summed by a warp (lane l takes l, l + 32, ...,
 *   then an xor butterfly) and the pieces in ascending order.  Totals over edges (the cost): tiles of 256 edges (warp
 *   butterflies, then the 8 warps in order); over images (the CG dot products): tiles of 32 images (a butterfly); the
 *   tile partials lane-strided in ascending order, then a butterfly.  The largest step is a max (exact).
 * - Launches: 1 kernel launch (cs_launch_count) whatever the sizes and iteration counts: one cooperative kernel (a
 *   resident wave, SMs x occupancy CTAs of 256 threads) runs the whole loop with grid barriers between its phases, after
 *   a cub sort of the incidences (not counted).  The call synchronises with the host once.  Scratch, in the per-device
 *   context: 216 bytes per image (its state), 32 per image and per 256 incidences (the pieces), 168 per edge (its state,
 *   final angle and the four sort arrays), 24 per iteration, plus the sort storage; pinned, the same tables.
 * - CS_E_ARG, before any CUDA call, naming the argument: numImages outside [1, 2^24], numEdges outside [0, 2^26],
 *   refImage outside [0, numImages), maxIterations outside [0, 1000], maxLinearIterations outside [1, 10000], linearTol
 *   not in (0, 1), sigmaDeg not in [0, 180], maxAngleDeg not in (0, 180], NULL edges, Rrel or weights with
 *   numEdges > 0, NULL R_out or cost_out, edges[e] with an image outside [0, numImages) or joining an image to itself,
 *   an Rrel[e] that is not finite or not a rotation (|R^T R - I| entries or |det R - 1| above 1e-6), weights[e] not
 *   finite or not > 0, and an output (R_out, residuals_out, inlier_out, cost_out, trace_out) that overlaps another
 *   output or an input (one sweep over sorted ranges, before any edge is read).  numEdges == 0 returns 0 with R = I
 *   for refImage and NaN for every other image, zero costs and trace, stats {0, 0, 1, 0, 0, 0}, and makes no CUDA
 *   call. */
int cs_rotation_averaging(int numImages, const int *edges, int numEdges, const double *Rrel, const double *weights,
                          int refImage, int maxIterations, int maxLinearIterations, double linearTol, double sigmaDeg,
                          double maxAngleDeg, double *R_out, double *residuals_out, unsigned char *inlier_out,
                          double cost_out[2], double *trace_out, long long stats_out[6], double ms_out[2]);

/* Global positioning (GLOMAP's BATA residual on points; Zhuang et al., CVPR 2018): every camera centre and track point
 * at once, from the rotations of cs_rotation_averaging, from random starts, with one robust least-squares problem over
 * all observations.  It takes cs_bundle_adjust's images and tracks (sets, Ks, d_offsets, d_members, d_use) and returns
 * the t that cs_triangulate_tracks and cs_bundle_adjust take.
 * - Images: Rs[a] is a rotation, or all nine entries NaN (cs_rotation_averaging's output for an image it did not
 *   reach): such an image takes no part.  refImage's centre is held at 0.
 * - Observations: tracks, malformed tracks and valid members follow cs_bundle_adjust (the tr_member rule).  A member is
 *   used when it is valid, its image has a rotation, and d_use is NULL or d_use[m] != 0; a track with at least 2 used
 *   members takes part, and observation o runs over their used members in track order, then member order.
 * - Residual of observation o (image a, track k): v_o = R_a^T K_a^-1 (x, y, 1) normalised, in float64;
 *   r_o = v_o - s_o (X_k - c_a).  Unknowns: the centres c_a of the images with a used observation (but refImage), the
 *   points X_k of the participating tracks, and one scale s_o per observation, kept >= 1e-6 (s <- max(s + ds, 1e-6)).
 * - Loss on |r_o|^2 as cs_bundle_adjust_intrinsics' (loss 0 trivial, 1 soft-L1, 2 Cauchy, scale c = lossScale, cost
 *   c^2 rho(|r|^2 / c^2), no 1/2), linearised by its corrector: r and every Jacobian block scaled by sqrt(rho').
 * - Start: c_a and X_k drawn uniform in [-1, 1)^3: component j of item i of kind q (0 centres, 1 points) is
 *   2 u - 1, u = (splitmix64(seed + 0x9E3779B97F4A7C15 ((q 2^32 + i) 3 + j)) >> 11) 2^-53; c_ref = 0; every s = 1.
 *   Two calls with one seed give the same bytes.
 * - LM: cs_bundle_adjust's rules (H + lambda D, D = diag(H) clamped to [1e-6, 1e32], taken before any elimination;
 *   lambda from 1e-3, /10 on accept, x10 on reject; accept when the solve succeeded and the cost decreased; stop after
 *   maxIterations, after an accepted step with previous - new <= 1e-10 previous, or when lambda exceeds 1e16).
 * - Linear solve: with w2 = rho', d = X - c and h = w2 |d|^2 damped, each s_o is eliminated from its own 7 x 7 block,
 *   leaving per observation P_o = w2 s^2 (I - w2 d d^T / h) on (X, c) as [P, -P; -P, P] and the right-hand side
 *   beta_o = w2 s (r - w2 d (d.r) / h) on X (-beta_o on c).  Points: V*_k = sum P_o + lambda clamp(sum w2 s^2) I by
 *   Cholesky, b_X = sum beta_o.  Cameras: U*_a likewise over a's observations; S = U* - W V*^-1 W^T,
 *   b~_a = -sum beta_o + sum P_o V*_k^-1 b_X,k.  Block-Jacobi PCG from dc = 0 with 3 x 3 blocks
 *   U*_a - sum_o P_o V*_k^-1 (sum of P over track k's observations in image a), cs_bundle_adjust's CG and stop rules.
 *   Then dX_k = V*_k^-1 (b_X,k + sum_o P_o dc_a) and ds_o = w2 (d.r - s d.(dX - dc)) / h.  A pivot not > 0 anywhere
 *   rejects the step.
 * - Gauge: the scale is held by the damping during the loop.  After it, c and X are divided by
 *   scale = sqrt(mean |c_a|^2) over the images with a used observation (refImage's 0 included; summed in tiles of 32
 *   images, then the tile partials), or 1 when that is not > 0.
 * - Outputs: t_out [numImages][3] = -R_a c_a / scale, NaN for an image with no used observation or with NaN R.
 *   d_points [numTracks][3] = X_k / scale, NaN for a track that does not take part.  cost_out = {start, final};
 *   trace_out (may be NULL) [maxIterations][4] as cs_bundle_adjust's; stats_out (may be NULL): [0] well-formed tracks,
 *   [1] malformed tracks, [2] invalid members, [3] used observations, [4] tracks positioned, [5] images with a used
 *   observation, [6] LM iterations, [7] CG iterations.  Returns the accepted steps, or CS_E_*.
 * - Determinism and launches: cs_bundle_adjust's: 3 kernel launches whatever the sizes (count, fill, one cooperative
 *   kernel), fixed summation orders (per point its observations in order; per camera tiles of 256 sorted observations
 *   and pieces in ascending order; totals over tiles of 256 tracks or 32 cameras), no floating-point atomics.  Scratch:
 *   416 bytes per image (state) plus 152 per image and per 256 members (pieces), 176 per track, 200 per member, 36 per
 *   LM iteration, plus the cub storage; pinned, 416 bytes per image and 32 per LM iteration.
 * - CS_E_ARG, before any CUDA call, naming the argument: numImages outside [1, 2^24], numTracks or numMembers < 0, NULL
 *   sets, Ks or Rs, refImage outside [0, numImages), loss outside 0..2, lossScale not finite or not > 0, maxIterations
 *   outside [0, 1000], maxLinearIterations outside [1, 10000], linearTol not in (0, 1), NULL t_out or cost_out, NULL
 *   d_offsets or d_points with tracks, NULL d_members with members, misaligned buffers, a set with records and no
 *   pointer, an invalid Ks[a] (cs_verify_essential's rule), an Rs[a] neither a rotation nor all NaN, d_points
 *   overlapping d_offsets, d_members, d_use or any set's records, and t_out, cost_out or trace_out overlapping each
 *   other, Ks or Rs.  numTracks == 0 returns 0 with NaN t, zero costs, trace and statistics, and makes no CUDA call. */
int cs_global_positioning(const cs_match_set *sets, int numImages, const double *Ks, const double *Rs,
                          const int *d_offsets, int numTracks, const int *d_members, int numMembers,
                          const unsigned char *d_use, int refImage, unsigned long long seed, int loss, double lossScale,
                          int maxIterations, int maxLinearIterations, double linearTol, double *t_out,
                          double *d_points, double cost_out[2], double *trace_out, long long stats_out[8], double *ms);

/* ---- dense reconstruction: undistorted images, PatchMatch stereo, depth-map fusion ----
 * Images are device float32 grayscale: pixel (col, row) is at d_img[row * pitch + col] (pitch in floats, >= width)
 * and lies at (col, row) in the coordinates that K maps to, the coordinates of the extractor's record positions.
 * Cameras are cs_bundle_adjust's: Ks[a] [9] (cs_verify_essential's rule), Rs[a] [9] a rotation, ts[a] [3], with
 * X_c = R X + t.  Every call checks, with CS_E_ARG before any CUDA call and naming the argument: numImages outside
 * [1, 65536] (cs_undistort_images: [0, 65536]), NULL images (or Ks, Rs, ts) with images, a NULL or not 4-byte aligned
 * images[a].d_img, width or height outside [2, 4096], pitch < width, and an invalid Ks[a], Rs[a] (R^T R = I within
 * 1e-6, det R > 0) or non-finite ts[a].
 * The bilinear sample of an image at (u, v), in FP32: u and v are clamped to [0, W - 1] and [0, H - 1], x0 =
 * min((int)u, W - 2), fx = u - x0 (likewise y0, fy), a = fmaf(fx, I(x0 + 1, y0) - I(x0, y0), I(x0, y0)),
 * b = fmaf(fx, I(x0 + 1, y0 + 1) - I(x0, y0 + 1), I(x0, y0 + 1)), and the sample is fmaf(fy, b - a, a). */
typedef struct {
  const float *d_img;
  int width, height, pitch;
} cs_image;

/* One depth map: image ref seen from the images sources[0 .. numSources) (a host array).  d_depth [H][W],
 * d_normal [H][W][3] (the normal in ref's camera frame) and d_cost [H][W] are dense device float arrays of ref's size.
 * An image is the ref of at most one job, so every random draw is keyed by the image and a job's maps do not depend
 * on the batch it is in. */
typedef struct {
  int ref;
  const int *sources;
  int numSources;
  float depthMin, depthMax;
  float *d_depth;
  float *d_normal;
  float *d_cost;
} cs_stereo_job;

/* Undistortion of whole images under cs_bundle_adjust_intrinsics' radial model: d_out[a] (device, dense
 * width x height floats) is images[a] as the pinhole camera Ks[a] would see it.  Size and K are kept.
 * - Output pixel (x, y), in float64: b = (y - K5) / K4, a = (x - K2 - K1 b) / K0, s = 1 + k1 r^2 + k2 r^4 with
 *   r^2 = a^2 + b^2 (the forward model of cs_undistort_records, in closed form), u = K0 a s + K1 b s + K2 and
 *   v = K4 b s + K5, rounded to float; the output is the bilinear sample of images[a] at (u, v), or 0 when (u, v) is
 *   outside [0, W - 1] x [0, H - 1] (counted in outside_out[a], may be NULL).  dists [numImages][2] (k1, k2) may be
 *   NULL (all zero: the input itself inside a 1-pixel border, where the position may round just outside or
 *   fx or fy = 1 may round the lerp).
 * - One kernel launch (cs_launch_count) for all images, whatever their sizes; the call synchronises once; *ms (may be
 *   NULL) gets its event time.  numImages == 0 makes no CUDA call.
 * - CS_E_ARG, before any CUDA call: the image and camera checks above (Rs and ts are not taken), a non-finite
 *   dists[a], NULL d_out, a NULL or not 4-byte aligned d_out[a], and an overlap of d_out[a] with another output or any
 *   image (one sweep over sorted ranges). */
int cs_undistort_images(const cs_image *images, int numImages, const double *Ks, const double *dists,
                        float *const *d_out, long long *outside_out, double *ms);

/* PatchMatch stereo (Bleyer et al., BMVC 2011) with red-black propagation (Gipuma, Galliani et al., ICCV 2015): a
 * depth, a normal and a cost for every pixel of every job's ref image, all jobs in one call.
 * - Hypothesis at pixel p = (x, y) of ref r: depth z along the camera axis and a unit normal n (ref camera frame) that
 *   faces the ray, n . ray < 0 with ray = Kinv (x, y, 1), Kinv = K_r^-1 in float64.  Its plane passes through X = z ray.
 * - Tables, on the host in float64 and rounded to float once: per source s of a job, A_s = K_s R_sr Kinv and
 *   b_s = K_s t_sr with R_sr = R_s R_r^T, t_sr = t_s - R_sr t_r.  Homography of h into s, in float64 from those floats
 *   and the float hypothesis, then rounded to float: m = (Kinv^T n) / (z (n . ray)), H_s = A_s + b_s m^T.
 * - View cost of h in s: the window is the (2 windowRadius / windowStep + 1)^2 offsets (i, j) in steps of windowStep
 *   from -windowRadius to windowRadius, rows j outer, columns i inner.  Reference sample R_ij = ref(clamp(x + i),
 *   clamp(y + j)) at integer positions; q = H_s (x + i, y + j, 1) in FP32, source sample S_ij = the bilinear sample of
 *   s at (q0 / q2, q1 / q2).  The view is invalid, and costs 2, when q2 <= 0 for some sample, when the centre's
 *   (u, v) lies outside [0, W_s - 1] x [0, H_s - 1], or when either window's variance is below 1 (grey levels^2).
 *   Otherwise, in FP32 in the window order, with the centre samples R_00 and S_00 taken first: d = R_ij - R_00,
 *   e = S_ij - S_00, sums of d, e, d^2, e^2 and d e (each by fmaf for the products); mean = sum / N, var = sum of
 *   squares / N - mean^2, cov = sum de / N - mean_d mean_e, and cost = 1 - cov / sqrtf(var_d var_e) clamped to [0, 2].
 *   Against the same view cost in float64 (from the same float H_s), an FP32 cost differs by at most 2e-3 when no
 *   decision above lies within 1e-3 of its threshold (a relative 1e-3 for the variance floor).
 * - Aggregated cost of h: the mean of its topK smallest view costs, summed in ascending order.
 * - Draws: u(slot) = (splitmix64(seed + 0x9E3779B97F4A7C15 c) >> 11) 2^-53 with the counter
 *   c = ((ref 2^24 + y W + x) 64 + iteration) 16 + slot.  A random hypothesis takes u(s0) for the depth, uniform in
 *   inverse depth: 1 / z = 1 / depthMax + u (1 / depthMin - 1 / depthMax), and u(s0 + 1 .. s0 + 3) for the normal,
 *   normalise(2 u - 1), negated when n . ray > 0 (-ray / |ray| when n . ray = 0 or the draw is 0).  Every value
 *   derived from draws is computed in float64 from the float state and rounded to float once.
 * - Start (iteration 0): every pixel takes the random hypothesis of slot 0 and its aggregated cost.
 * - Iteration k = 1 .. numIterations, rho = 2^-k: a half-step over the pixels with x + y even, then one over the odd
 *   ones.  A pixel's candidates, in this order, from the state at the start of the half-step:
 *   1. propagation from the neighbours at (-1, 0), (1, 0), (0, -1), (0, 1), (-5, 0), (5, 0), (0, -5), (0, 5) (all of the
 *      other colour): the neighbour's plane, through z_q Kinv (x_q, y_q, 1), met by p's ray: z = (n_q . X_q) / (n_q . ray)
 *      with n_q; skipped when q is off the image, when n_q . ray >= 0, or when z (as float) is outside
 *      [depthMin, depthMax];
 *   2. the depth moved in inverse depth, 1 / z + rho (2 u(0) - 1) (1 / depthMin - 1 / depthMax) clamped to
 *      [1 / depthMax, 1 / depthMin], with the current normal;
 *   3. the current depth with the normal normalise(n + rho (2 u(1 .. 3) - 1)), negated to face the ray as above;
 *   4. both moves, with u(4) and u(5 .. 7);
 *   5. the random hypothesis of slot 8.
 *   The pixel keeps the candidate of strictly lowest aggregated cost: ties go to the current hypothesis, then to the
 *   earlier candidate.  A half-step reads the other colour and the pixel's own state only, so the maps are the state,
 *   and the result does not depend on the order in which pixels run: two calls give the same bytes, and a job's maps
 *   are the same bytes alone or in any batch.
 * - Outputs: every pixel ends with a finite hypothesis and its cost; cost 2 means no source supported it.
 *   stats_out [numJobs][3] (may be NULL): pixels, invalid view evaluations in the whole call, pixels whose final cost
 *   is 2.
 * - Launches: 2 + 2 numIterations kernel launches (cs_launch_count) for all jobs together (start, the half-steps, a
 *   final count); the call synchronises once; *ms (may be NULL) gets its event time.  Scratch in the per-device
 *   context: the image, job and source tables (264 bytes per image, 144 per job, 52 per source) and 24 bytes per job
 *   of counters; the same tables pinned.  numJobs == 0 makes no CUDA call.
 * - CS_E_ARG, before any CUDA call: the image and camera checks above, numJobs outside [0, 65536], NULL jobs with
 *   jobs, windowRadius outside [1, 7], windowStep outside [1, windowRadius] or not dividing windowRadius,
 *   numIterations outside [0, 32], and per jobs[p]: ref outside [0, numImages) or the ref of an earlier job,
 *   numSources outside [1, 32], NULL sources, a source outside [0, numImages), equal to ref or listed twice, topK
 *   outside [1, numSources], depthMin and depthMax not finite or not 0 < depthMin < depthMax, and NULL or not 4-byte
 *   aligned d_depth, d_normal or d_cost; then an overlap of a map with any other map or image (one sweep). */
int cs_patch_match_stereo(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
                          const cs_stereo_job *jobs, int numJobs, int windowRadius, int windowStep, int numIterations,
                          int topK, unsigned long long seed, long long *stats_out, double *ms);

/* A prior depth map of an image: d_depth [H][W] and d_normal [H][W][3], dense device floats of the image's size. */
typedef struct {
  const float *d_depth;    /* NULL: the image has no prior */
  const float *d_normal;   /* needed only for an image that is the ref of a job */
} cs_depth_prior;

/* PatchMatch stereo with geometric consistency (Schoenberger et al., ECCV 2016: COLMAP's second pass): every job's
 * maps again, each view's cost joined by a forward-backward reprojection error against that source's prior depth map.
 * Images, cameras, jobs and window are cs_patch_match_stereo's; the jobs' d_depth, d_normal and d_cost are outputs
 * only.  priors [numImages] are read only, and per image, so a call may refine some refs and read the priors of all.
 * - Geometric error of hypothesis h = (z, n) at pixel (x, y) of ref r in source s, in float64: X = z Kinv_r (x, y, 1);
 *   Y = R_sr X + t_sr (R_sr = R_s R_r^T, t_sr = t_s - R_sr t_r, from the double cameras); (u, v) = (K_s Y)_0,1 / Y_z;
 *   q = (floor(u + 0.5), floor(v + 0.5)); z_s the prior depth of s at q; X_s = z_s Kinv_s (u, v, 1) (the continuous
 *   (u, v), so a consistent pair gives an error near 0); Z = R_sr^T (X_s - t_sr); (u', v') = (K_r Z)_0,1 / Z_z;
 *   e = hypot(u' - x, v' - y) and g = (float) min(e, geomMaxError).  g = geomMaxError when Y_z <= 0 or Z_z <= 0, q lies
 *   outside s, s has no prior, or z_s is not finite or <= 0 (depth 0 masks a pixel out).
 * - View cost: fmaf(lambda, g, c_photo) with lambda = (float) geomWeight, c_photo the photometric view cost (2 for an
 *   invalid view, which still carries its g).  Aggregation (the mean of the topK smallest, in ascending order) and
 *   selection are cs_patch_match_stereo's.
 * - Start: each pixel takes its ref's prior (z_p, n_p) bit for bit when z_p is in [depthMin, depthMax], n_p is finite,
 *   n_p . ray < 0 and | |n_p| - 1 | <= 1e-3 (in float64 from the floats); otherwise the random hypothesis of counter
 *   iteration 32, slot 0.  Either way it gets its combined cost.
 * - Iterations k = 1 .. numIterations: cs_patch_match_stereo's candidate list, order and rho = 2^-k, with the draws at
 *   counter iteration 32 + k, so the two passes' draws differ under the same seed.  The priors are inputs, never state:
 *   two calls give the same bytes, and a job's maps are the same alone or in any batch given the same priors.
 * - stats_out [numJobs][5] (may be NULL): pixels, invalid view evaluations, pixels whose final cost is >= 2,
 *   photometrically valid view evaluations whose g is geomMaxError, pixels started from a random hypothesis.
 * - Launches: 2 + 2 numIterations (start, the half-steps, a final count); the call synchronises once; *ms (may be
 *   NULL) gets its event time.  Scratch: cs_patch_match_stereo's tables, plus 112 bytes per source (R_sr, t_sr, the
 *   source's prior and size) and 16 per job (the ref's prior), and 48 bytes per job of counters; the same pinned.
 *   numJobs == 0 makes no CUDA call.
 * - CS_E_ARG, before any CUDA call: cs_patch_match_stereo's checks, but numIterations outside [0, 31]; NULL priors with
 *   jobs; a job whose ref has a NULL prior d_depth or d_normal; a prior pointer that is not 4-byte aligned;
 *   geomWeight not finite or < 0; geomMaxError not finite or <= 0; then an overlap of a map with any other map, any
 *   prior or any image (one sweep; priors may overlap each other and the images). */
int cs_patch_match_stereo_geometric(const cs_image *images, int numImages, const double *Ks, const double *Rs,
                                    const double *ts, const cs_depth_prior *priors, const cs_stereo_job *jobs,
                                    int numJobs, int windowRadius, int windowStep, int numIterations, int topK,
                                    double geomWeight, double geomMaxError, unsigned long long seed,
                                    long long *stats_out, double *ms);

/* Fusion of the depth maps of cs_patch_match_stereo into one point cloud (COLMAP's stereo_fusion, as a parallel rule
 * whose order follows from the values): jobs, their maps and the images as that call left them.
 * - Pixel p = (x, y) of job a (image a = jobs[.].ref) with cost <= maxCost back-projects to X_p = R_a^T (z Kinv_a
 *   (x, y, 1) - t_a) with world normal R_a^T n.  A source b of job a that is itself the ref of a job is consistent
 *   when, in float64: Y = R_b X_p + t_b has Y_z > 0; q = (floor(u + 0.5), floor(v + 0.5)) for (u, v) = K_b Y / Y_z
 *   lies in b; cost_b(q) <= maxCost; |z_b(q) - Y_z| <= maxDepthError Y_z; the world normals of p and q have a dot
 *   product >= cos(maxNormalErrorDeg); and q back-projected with z_b(q) projects into a within maxReprojError pixels
 *   of (x, y).
 * - p emits a point when it has at least minConsistent consistent views and none of them has an image index below a,
 *   so a surface point is emitted by the lowest-indexed image that sees it consistently.  A duplicate can still
 *   appear when source lists are asymmetric: b emits its own point for q when a is not a source of b.
 * - The point: position the mean of X_p and the consistent back-projections, normal the normalised sum of the world
 *   normals, intensity the mean of image a at p and each consistent image at q, summed in float64 in source-list order
 *   after p's own; d_source = {a, y W + x}.  Outputs d_xyz [][3], d_normal [][3], d_intensity [] (float) and d_source
 *   [] (int2), in ascending (a, pixel) order, written by a flag kernel and a count-scan-write kernel (ordered_list.cuh),
 *   at most maxPoints (the prefix of the full list).
 * - Returns the number of points in the full list, or CS_E_*.  stats_out (may be NULL): [0] that number, [1] the
 *   points written.  2 kernel launches; the call synchronises once; *ms (may be NULL) gets its event time.  Scratch:
 *   cs_patch_match_stereo's tables and counters, plus, on the device only, the list's words (4 bytes per 32 pixels,
 *   4 per 1024).
 *   numJobs == 0 returns 0 and makes no CUDA call.
 * - CS_E_ARG, before any CUDA call: cs_patch_match_stereo's image, camera and job checks (topK aside), the pixels of
 *   all jobs above 2^31 - 1, maxCost not in [0, 2], minConsistent outside [1, 32], maxReprojError, maxDepthError not
 *   finite or not > 0, maxNormalErrorDeg not in (0, 180], maxPoints < 0, NULL or not 4-byte aligned d_xyz, d_normal,
 *   d_intensity or d_source (8-byte) with maxPoints > 0; and an overlap of an output with any other output, map or
 *   image (one sweep). */
int cs_fuse_depth_maps(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
                       const cs_stereo_job *jobs, int numJobs, float maxCost, int minConsistent, double maxReprojError,
                       double maxDepthError, double maxNormalErrorDeg, float *d_xyz, float *d_normal,
                       float *d_intensity, int *d_source, int maxPoints, long long stats_out[2], double *ms);

/* Poisson surface reconstruction (Kazhdan, Bolitho & Hoppe, SGP 2006) of an oriented point cloud, such as the output
 * of cs_fuse_depth_maps, on a dense regular grid: a closed, oriented triangle mesh.  The grid is dense, so the
 * resolution is capped at 512 cells per axis (no octree); there is no screening term and no per-point weight.
 * - Used points: d_xyz [numPoints][3], d_normal [numPoints][3] (device floats, outward normals of any length) and
 *   d_intensity [numPoints] (may be NULL).  Point i is used when its six coordinates are finite and |n| > 0; its unit
 *   normal n^ = n / |n| is computed in float64 from the floats.
 * - Grid: N = 2^depth cells per axis, (N + 1)^3 nodes, node (i, j, k) at index (k (N + 1) + j) (N + 1) + i.  In float64:
 *   lo, hi the component-wise min and max of the used xyz (exact in any order), c = (lo + hi) / 2, E = max(hi - lo),
 *   L = max(scale, N / (N - 8)) E (at least 4 cells of margin on every side), h = L / N, o = c - L / 2, and a point's
 *   grid coordinate g = (p - o) / h.  No used point, or E = 0: status 1, no triangles, info_out zero, chi zero.
 * - Splat (a gather, no atomics): the used points sorted by cell floor(g) (index (c_z N + c_y) N + c_x) with a stable
 *   radix sort, so ties keep the point order.  Node q sums over the points of its (up to 8) incident cells, cells in
 *   ascending index and points in sorted order, with weight w = prod_a (1 - |g_a - q_a|): V(q) = sum w n^,
 *   D(q) = sum w and, with intensities, S(q) = sum w I, each accumulated in float64 and rounded to float once.
 * - System: chi = 0 on the boundary nodes; at each interior node 6 chi_q - sum of the 6 neighbours = b_q with
 *   b_q = (h / 2) sum_a (V_a(q + e_a) - V_a(q - e_a)) (h^2 times the central-difference divergence), in float64 from
 *   the float V, rounded to float, summed as (x + y) + z.  With outward normals chi is larger inside.
 * - Solve: CG from chi = 0 preconditioned by one geometric-multigrid V-cycle (MGPCG; McAdams, Sifakis & Teran, SCA
 *   2010).  Vectors are float32; every dot product and norm is float64.  Levels of n = N, N / 2, ..., 4 cells, each with
 *   the 7-point operator above (6 x - neighbours, boundary 0).  On a level, from x = 0: 2 pairs of red-black
 *   Gauss-Seidel half-sweeps (red: (i + j + k) even; x = (f + neighbours) / 6 in float), the residual t = f - A x, the
 *   coarse right-hand side (1/2) P^T t (P trilinear prolongation: the 27 fine nodes 2Q + d weigh prod (1 - |d_a| / 2)),
 *   the V-cycle on the coarser level, x += P x_c, then 2 pairs of black-red half-sweeps.  The coarsest level (4 cells)
 *   runs 8 red-black pairs then 8 black-red pairs.  The sweep sequence is a palindrome and the restriction is a
 *   multiple of P^T, so the preconditioner is symmetric positive definite.  CG: r = b, z = M r, p = z; per iteration
 *   q = A p, alpha = r.z / p.q (stop when p.q is not > 0), chi += alpha p, r -= alpha q (each in float64 from the
 *   floats, rounded to float), then it stops when r.r <= tol^2 b.b (the recurrence residual) or after maxIterations;
 *   else z = M r, beta = r.z(new) / r.z(old), p = z + beta p.  alpha, beta and the stop test are computed on the
 *   device.  After the loop the true relative residual |b - A chi| / |b| (0 when b = 0) in float64 from the floats.
 * - Iso-value: tau the mean over the used points of chi trilinear at g (cell clamp(floor(g), 0, N - 1), corners z outer,
 *   x inner), the mean density the same of D, summed in float64 in sorted order.  tau <= 0 (inconsistent normals, b = 0,
 *   or an open surface seen from one side, whose points lie where chi < 0): status 2, no triangles.
 * - Extraction (marching tetrahedra, Doi & Koide 1991, on the Freudenthal split: no case table, no ambiguous case): a
 *   node is inside when (double) chi_q >= tau.  The lattice edges of node q go to q + delta for delta in the order
 *   (1,0,0), (0,1,0), (0,0,1), (1,1,0), (1,0,1), (0,1,1), (1,1,1); edge id 7 index(q) + direction.  Every edge whose
 *   ends differ in inside has a vertex at t = (tau - chi_a) / (chi_b - chi_a) (float64 from the floats), position
 *   o + h (q + t delta) rounded to float; vertices are listed in ascending edge id.  Cell q0 splits into 6 tetrahedra,
 *   one per axis permutation pi in lexicographic order, with corners q0, q0 + e_pi1, q0 + e_pi1 + e_pi2, q0 + (1,1,1).
 *   One or three inside corners: one triangle on the three edges of the lone corner a, vertices in the order of the
 *   other corners along the chain.  Two inside corners a, b and two outside c, d (chain order): the quad
 *   (ac, ad, bd, bc), split along the diagonal ac-bd into (ac, ad, bd), (ac, bd, bc).  Orientation, decided on the
 *   edge midpoints: (v1 - v0) x (v2 - v0) points to the outside corners (else the cycle is reversed after its first
 *   vertex).  Triangles are listed in ascending (cell, tetrahedron, k).  Since tau > 0 and the boundary is 0, the mesh
 *   is combinatorially a closed, oriented 2-manifold for any values; exact ties (t = 0) give zero-area triangles.
 * - Trim (COLMAP's trim on a dense grid): a vertex's density is D_a + t (D_b - D_a) in float64; a triangle with a vertex
 *   of density < trim x mean density is dropped; vertices no kept triangle uses are dropped, the rest keep their
 *   order and the triangles are renumbered.  trim = 0 drops nothing.
 * - Vertex intensity (with d_intensity and d_vertexIntensity): (S_a + t (S_b - S_a)) / (D_a + t (D_b - D_a)), 0 when
 *   the denominator is 0.
 * - Outputs: d_vertices [][3] float, d_triangles [][3] int32 (indices into the full trimmed vertex list, so a written
 *   triangle may name a vertex at or beyond maxVertices) and d_vertexIntensity [], each the prefix of its full list
 *   (at most maxVertices or maxTriangles entries).  d_chi [(N + 1)^3] (may be NULL): chi.  info_out [7] (may be NULL):
 *   {o_x, o_y, o_z, h, tau, mean density, true relative residual}.  stats_out [10] (may be NULL): used points, refused
 *   points, CG iterations, vertices and triangles before trimming, vertices and triangles after trimming (the full
 *   counts), vertices written, triangles written, status (0 ok, 1 no used point or zero extent, 2 tau <= 0, 3 not
 *   converged: the mesh is still extracted).  Returns the full trimmed triangle count, or CS_E_*.
 * - Determinism: no floating-point atomics (integer atomics for the box, the cell histogram and the kept-vertex bits,
 *   whose results do not depend on order); totals over nodes or points sum tiles of 2048 items (a thread adds items
 *   thread + 256 m in order, then warp butterflies and the warps in order), then groups of 256 tile partials the same
 *   way, then the group partials (lane-strided in ascending order and a butterfly): the order depends on N and the
 *   used count only, so two calls give the same bytes.
 * - Launches: 10 kernel launches (cs_launch_count) whatever the depth and the data (box, keys, points, splat,
 *   right-hand side, one cooperative solve kernel, two counts, vertices, triangles), plus cub's sort and scans (not
 *   counted).  The lists are written by per-block counts, cub::DeviceScan and a write pass.  The call synchronises
 *   once; *ms (may be NULL) gets its event time.
 * - Scratch, allocated on the call's stream and freed before it returns (no grid-sized memory is kept): 4 x 7 bytes
 *   per node (8 with intensities: chi, r, b, the three V components reused as z, p, q, D, S), 12 per node of every
 *   coarser level, 1 per node (kept-vertex bits), 64 per block of 256 nodes, 68 bytes per point (64 without
 *   intensities), the sort and scan storage: about 4.3 GB at depth 9 (513^3 nodes) with intensities.
 * - CS_E_ARG, before any CUDA call, naming the argument: numPoints outside [0, 2^30], depth outside [4, 9], scale not
 *   finite or outside [1, 4], maxIterations outside [1, 1000], tol not in (0, 1), trim not finite or < 0, maxVertices
 *   or maxTriangles < 0, NULL or not 4-byte aligned d_xyz or d_normal with numPoints > 0, d_vertices with
 *   maxVertices > 0, d_triangles with maxTriangles > 0, a misaligned d_intensity, d_vertexIntensity or d_chi, one of
 *   d_intensity and d_vertexIntensity given without the other, and an output (d_vertices, d_vertexIntensity,
 *   d_triangles, d_chi) that overlaps another output or an input (one sweep over sorted ranges). */
int cs_poisson_mesh(const float *d_xyz, const float *d_normal, const float *d_intensity, int numPoints, int depth,
                    double scale, int maxIterations, double tol, double trim, float *d_vertices,
                    float *d_vertexIntensity, int maxVertices, int *d_triangles, int maxTriangles, float *d_chi,
                    double info_out[7], long long stats_out[10], double *ms);

/* Screened Poisson surface reconstruction (Kazhdan & Hoppe, ACM TOG 2013) with a Neumann boundary, on the same dense
 * grid as cs_poisson_mesh: a mesh of open surfaces seen from one side (a terrain, a facade, a fused stereo scene) as
 * well as closed ones.  The arguments are cs_poisson_mesh's plus pointWeight (alpha), after scale.
 * - Used points, grid, sort, splat, V, D, S and intensities: exactly as in cs_poisson_mesh (the same kernels).
 * - Operator (Neumann boundary): the graph Laplacian on all (N + 1)^3 nodes, (L x)_q = deg_q x_q - sum of the in-grid
 *   neighbours (deg_q in [3, 6]).
 * - Right-hand side: the divergence of the edge field g(q -> q + e_a) = (h / 2)(V_a(q) + V_a(q + e_a)): b_q = sum over
 *   the in-grid edges leaving q of g - sum over those entering q of g.  In float64 from the float V, per axis
 *   V_a(q + e_a) - V_a(q - e_a) with both neighbours (the central difference of cs_poisson_mesh), V_a(q) + V_a(q + e_a)
 *   at a low face, -(V_a(q - e_a) + V_a(q)) at a high face, then (h / 2)((x + y) + z) rounded to float.  Sum b = 0 in
 *   exact arithmetic.
 * - Screening: A = L + omega sum_p B_p B_p^T, where B_p holds point p's trilinear weights prod_a (1 - |g_a - q_a|) at
 *   the 8 corners of its cell clamp(floor(g), 0, N - 1) (z outer, x inner).  The target is 0, so b has no screening
 *   term.  omega = pointWeight / mean density, the mean density computed before the solve exactly as info_out[5] of
 *   cs_poisson_mesh.  Since 1^T L = 0, 1^T b = 0 and sum_c B_p(c) = 1, the mean of chi at the points is 0 in exact
 *   arithmetic.
 * - Solve: cs_poisson_mesh's CG with A p as L p in float plus (float) S p, where u_p = omega B_p^T p over the sorted
 *   points (float64 from the floats), a grid barrier, then (S p)_q = sum B_p(q) u_p over the points of q's (up to 8)
 *   cells, cells in ascending index and points in sorted order, in float64.  The preconditioner is one V-cycle with
 *   cs_poisson_mesh's schedule (2 pairs, 8 coarsest pairs, levels down to 4 cells, restriction (1/2) P^T) on the level
 *   operators L_l + diag(s_l) over every node, boundary included: the half-sweep x = (f + in-grid neighbours) /
 *   (deg + s_q), the residual f - ((deg + s_q) x - neighbours), restriction and prolongation over the in-grid nodes.
 *   s_l is the diagonal of the exact coarse screening (1/2) P^T S_(l-1) P = (omega / 2^l) sum B^l_p B^l_p^T at the
 *   level-l coordinates g / 2^l: s_l(Q) = (omega / 2^l) sum (B^l_p(Q))^2 over the fine cells of Q's support in
 *   ascending index, in float64, rounded once (level 0 a thread per node; coarser levels a warp per node, lane j
 *   summing rows of cells j, j + 32, ... then a butterfly).  The V-cycle stays symmetric positive definite.  The true
 *   relative residual uses the same A in float64 from the floats.
 * - Iso-value: tau is the mean of chi at the used points, as in cs_poisson_mesh; it is near 0 and its sign means
 *   nothing, so status 2 never occurs.  Extraction (inside: chi >= tau), trim, vertex intensity, outputs and their
 *   order: as in cs_poisson_mesh (the same kernels).  Without trimming the mesh is an oriented 2-manifold whose
 *   boundary edges all lie on the grid's faces.
 * - info_out [8] (may be NULL): cs_poisson_mesh's 7 entries, then omega.  stats_out [10]: cs_poisson_mesh's layout;
 *   status 0 ok, 1 no used point or zero extent, 3 not converged (the mesh is still extracted).
 * - Determinism: no floating-point atomics; every sum has a fixed order (above, and cs_poisson_mesh's totals).
 * - Launches: 10 kernel launches whatever the depth and the data (box, keys, points, splat, right-hand side, one
 *   cooperative solve kernel, two counts, vertices, triangles), plus cub's sort and scans (not counted).
 * - Scratch: cs_poisson_mesh's, plus 4 bytes per node of every level (s_l), 4 per node (cell starts the solve keeps)
 *   and 8 per point (u): about 5.5 GB at depth 9 with intensities.
 * - CS_E_ARG, before any CUDA call, naming the argument: pointWeight not finite or outside (0, 1000], then every check
 *   of cs_poisson_mesh (the same ranges and the same overlap sweep). */
int cs_poisson_mesh_screened(const float *d_xyz, const float *d_normal, const float *d_intensity, int numPoints,
                             int depth, double scale, double pointWeight, int maxIterations, double tol, double trim,
                             float *d_vertices, float *d_vertexIntensity, int maxVertices, int *d_triangles,
                             int maxTriangles, float *d_chi, double info_out[8], long long stats_out[10], double *ms);

/* Mesh simplification: Garland & Heckbert's quadric error metric edge collapse (SIGGRAPH 1997) in a sequence of
 * parallel passes, each collapsing an independent set of edges chosen by values alone (after Papageorgiou & Platis
 * 2015, with a stricter independence rule), so the result is deterministic.  The inputs are device buffers in the layout
 * cs_poisson_mesh writes, so the two calls chain without a copy: d_vertices [numVertices][3] float,
 * d_vertexIntensity [numVertices] (may be NULL), d_triangles [numTriangles][3] int32.  All arithmetic below is float64,
 * each product, sum, quotient and square root rounded once, in the order written (no contraction).
 * 1. Input: status 2 and nothing written when a triangle index lies outside [0, numVertices), a triangle repeats a
 *    vertex, or a vertex some triangle uses has a non-finite coordinate.  A vertex is frozen (no edge at it ever
 *    collapses) when its faces do not form a single fan (one cycle or one open chain), or an edge at it has more than
 *    two faces or two faces that traverse it in the same direction.  Frozen status is computed once from the input;
 *    the link condition (rule 4) keeps every other vertex manifold.
 * 2. Quadrics (10 entries, the upper triangle of the 4x4 matrix row-major; plane p = (n, d) adds w (p_i p_j) to entry
 *    (i, j)): a face with n = (p1 - p0) x (p2 - p0) (x, y, z components as a1 b2 - a2 b1, a2 b0 - a0 b2,
 *    a0 b1 - a1 b0; dot products (x + y) + z), |n| = sqrt(n.n) > 0 adds its unit plane n / |n|, d = -(n^.p0) with
 *    w = area = |n| / 2; a boundary edge a -> b of such a face adds the plane of unit normal m / |m|, m = (b - a) x n^,
 *    through a, with w = boundaryWeight |b - a|^2.  A vertex that is not frozen sums its faces in ascending index, then
 *    the boundary edges at it of those faces in (face, corner) order, and the area sum A of its faces.  A collapse of
 *    (u, v) gives Q_u + Q_v and A_u + A_v.
 * 3. Edges: an undirected edge is identified by one canonical corner 3t + k (t the input index of its face; the edge
 *    runs from corner k to corner k + 1 mod 3): for an interior edge the corner with a < b, for a boundary edge its
 *    only corner; s(id) (rule 5) breaks every tie.  For Q = Q_u + Q_v = (a11 a12 a13 b1 a22 a23 b2 a33 b3 c) the position is
 *    the minimiser -A^-1 b by Cramer's rule when det(A) = (a11 (a22 a33 - a23^2) - a12 (a12 a33 - a23 a13)) +
 *    a13 (a12 a23 - a22 a13) > 1e-6 a11 a22 a33 (scale-invariant), else the best of u, v and the midpoint (ties to u,
 *    then v).  cost = ((a11 x0^2 + a22 x1^2) + a33 x2^2) + 2 ((a12 x0 x1 + a13 x0 x2) + a23 x1 x2) +
 *    2 ((b1 x0 + b2 x1) + b3 x2) + c, clamped at 0; the error is cost / A (0 when A = 0 and cost = 0, else infinite
 *    when A = 0), a mean squared distance.  An edge is admissible when its error is finite and sqrt(error) <= maxError.
 * 4. Validity: neither end frozen; the link condition (Dey et al. 1999): every vertex adjacent to both u and v is an
 *    apex of a face on uv, an interior edge whose apexes w1, w2 lie in a face with u and in a face with v is refused
 *    (the tetrahedron), an interior edge may not join two boundary vertices, and a boundary edge whose apex meets u and
 *    v by boundary edges is refused; every surviving face of u and v with n.n > 0 keeps n_old . n_new > 0 (no flip,
 *    and no face goes from area > 0 to area 0).
 * 5. Pass: a candidate's key is (float(error) bits << 32) | s(edge id), float() rounding to nearest, with the
 *    bijection s(i) = m ^ (m >> 16), m = i * 0x9E3779B1 mod 2^32: keys are unique, and equal errors (a flat region)
 *    are not ordered along the input's raster, where only one edge per pass would hold the minimum of its rings.  Of
 *    the C admissible candidates only the ceil(C/2) with the smallest keys compete (f = 1/2, chosen by a sweep,
 *    DESIGN.md section 9); each writes atomicMin of its key
 *    onto every vertex of the faces of u and of v (the closed 1-rings), and is selected when all of them hold its key.
 *    Selected edges have disjoint closed neighbourhoods, so their collapses do not interact.
 * 6. Collapse: the lower index u survives at the position, v maps to u; faces holding both are dropped, the others
 *    keep their cyclic order.  Intensity: I_u + t (I_v - I_u) with t = ((x - p_u).(p_v - p_u)) / |p_v - p_u|^2 clamped
 *    to [0, 1] (0 when p_u = p_v), rounded to float.  Vertex ids stay those of the input.
 * 7. Stop: before a pass, when T <= targetTriangles (status 0) or after 1000 passes (status 3); a pass with no
 *    admissible candidate ends the call (status 1).  In a pass that would cross the target only the selected edges
 *    with the smallest keys are applied, the fewest whose dropped faces reach T - targetTriangles, so the result ends
 *    at the target or one below.  Status 2: invalid input, nothing written.
 * 8. Outputs: d_outVertices [][3] float (the vertices the surviving triangles use, in ascending input index),
 *    d_outIntensity [] (with d_vertexIntensity), d_outTriangles [][3] (the survivors in ascending input index,
 *    renumbered into the full vertex list), each the prefix of its full list (at most maxOutVertices or
 *    maxOutTriangles entries).  info_out [1] (may be NULL): the largest applied sqrt(cost / A).  stats_out [9] (may be
 *    NULL): input triangles, frozen vertices, passes (that applied a collapse), collapses, full vertex and triangle
 *    counts, vertices and triangles written, status.  Returns the full triangle count, or CS_E_*.  numTriangles == 0
 *    returns 0 (status 0) and makes no CUDA call.
 * - Launches (cs_launch_count): 4 setup kernels (validate, init, corner keys, frozen and quadrics; 1 when the input is
 *   invalid), 8 per pass (candidates, threshold, scatter, select, collapse, face count, face write, corner keys), 4 in
 *   a final pass that finds no admissible edge, 1 more in a pass that crosses the target, and 4 output kernels; plus
 *   cub's sorts and scans (not counted).  The host reads a few words after the input check and after each pass's
 *   selection (one synchronise each); *ms (may be NULL) gets the event time of the whole call.
 * - Scratch, allocated on the call's stream and freed before it returns: 212 bytes per triangle (two triangle lists and
 *   input indices, corner keys and values and their sorted copies, candidate and selected keys and their sorted
 *   copies, dropped-face counts and their scan) and 141 per vertex (float64 position, quadric and area, intensity,
 *   frozen flag, remap, output index, minimum key, face counts and starts), plus cub's storage.
 * - CS_E_ARG, before any CUDA call, naming the argument: numVertices outside [0, 2^30], numTriangles outside [0, 2^29],
 *   targetTriangles < 0, maxError NaN or < 0 (inf allowed), boundaryWeight not finite or < 0, maxOutVertices or
 *   maxOutTriangles < 0, NULL or not 4-byte aligned d_vertices with numVertices > 0, d_triangles with
 *   numTriangles > 0, d_outVertices with maxOutVertices > 0, d_outTriangles with maxOutTriangles > 0, a misaligned
 *   d_vertexIntensity or d_outIntensity, one of them given without the other, and an output (d_outVertices,
 *   d_outIntensity, d_outTriangles) that overlaps another output or an input (one sweep over sorted ranges). */
int cs_simplify_mesh(const float *d_vertices, const float *d_vertexIntensity, int numVertices, const int *d_triangles,
                     int numTriangles, int targetTriangles, double maxError, double boundaryWeight,
                     float *d_outVertices, float *d_outIntensity, int maxOutVertices, int *d_outTriangles,
                     int maxOutTriangles, double info_out[1], long long stats_out[9], double *ms);

/* Mesh cleaning: the clean-up between meshing and the later mesh stages (OpenMVS's Mesh::Clean), in one deterministic
 * call.  It drops degenerate, duplicate, long-edge and non-manifold-edge faces and small components, closes small holes
 * by ear cutting without new vertices, and optionally smooths.  The inputs and outputs are in cs_simplify_mesh's
 * layout, so the calls chain without a copy: d_vertices [numVertices][3] float, d_vertexIntensity [numVertices] (may
 * be NULL), d_triangles [numTriangles][3] int32.  All arithmetic below is float64 from the float positions, each
 * product, sum, quotient and square root rounded once, in the order written (no contraction); n(a, b, c) =
 * (p_b - p_a) x (p_c - p_a) and dot products as in cs_simplify_mesh's rule 2.  Corner 3t + k starts the edge from corner
 * k to corner k + 1 mod 3.  The rules run in this order, each on the faces the rules before it keep:
 * 1. Input: cs_simplify_mesh's rule 1; status 2 and nothing written when it fails.
 * 2. (removeDegenerate) A face with n.n == 0 is dropped (degenerate), unless each of its three edges is held by another
 *    input face: such a face lies inside the surface (marching tetrahedra leaves them in closed meshes), and dropping
 *    it would open a flat slit that no allowed ear of rule 6 closes, so it stays.  Of the remaining faces with the same
 *    vertex set, in either orientation, the lowest index stays and the others are dropped (duplicate).
 * 3. (longEdgeFactor > 0) Over the distinct undirected edges of the kept faces, in ascending key (min << 32) | max,
 *    with length l = sqrt(d.d), d = p_max - p_min: N = sum 1, S1 = sum l and S2 = sum l l in coop.cuh's three-level
 *    order (tiles of 2048 positions of the sorted corner edge keys of all 3 numTriangles input corners, a value at the
 *    first position of each kept edge; groups of 256 tiles); m = S1 / N, s = sqrt(S2 / N - m m) (0 when
 *    not positive), threshold m + longEdgeFactor s.  A face with an edge longer than the threshold is dropped.
 * 4. (removeNonManifold) On an edge held by three or more kept faces, the two lowest-index faces stay and the others
 *    are dropped, all against the faces kept before the rule.  Dropping faces creates no new non-manifold edge, so one
 *    pass suffices.  Non-manifold vertices are not split: a vertex is counted as non-manifold when the corners at it
 *    of the faces kept after this rule form more than one fan, corners of two faces joining across an edge at the
 *    vertex held by exactly two of those faces.
 * 5. Faces join across edges held by exactly two kept faces; the components are built by union-find whose root is the
 *    lowest face.  With minComponentFaces > 1 or minComponentFraction > 0, a component is dropped when its face count
 *    n < minComponentFaces or n < minComponentFraction n_max (as float64), n_max the largest component's count.
 * 6. (maxHoleEdges > 0, at most 256) A kept face's corner edge a -> b held by no other kept face gives the boundary
 *    half-edge b -> a (the loop direction, so fill faces take their neighbours' orientation).  A half-edge's successor
 *    is the half-edge out of its end vertex when that vertex has exactly one boundary half-edge in and one out; the
 *    half-edges on a successor cycle form a loop that starts at its lowest vertex id (found by pointer jumping); the
 *    others lie on no loop.  A loop of L <= maxHoleEdges edges (L >= 3 always) is filled by ear cutting over its
 *    vertices r_0 .. r_{L-1} in loop order: with the reference normal N = sum_{i=1}^{L-2} n(r_0, r_i, r_{i+1}) summed
 *    in i order, the ear at position i of the current ring (prev, cur, next) is allowed when n(prev, cur, next).N > 0
 *    (no reflex and no zero-area ear), no kept face holds the edge {prev, next}, and no other ring vertex q has
 *    n(prev, cur, q).N > 0, n(cur, next, q).N > 0 and n(next, prev, q).N > 0 (inside the ear); of the allowed ears the one with the largest
 *    c = (u.w) / sqrt((u.u)(w.w)), u = p_prev - p_cur, w = p_next - p_cur (the smallest apex angle) is cut, ties to the
 *    lowest position; the face (prev, cur, next) is added and cur leaves the ring.  With three vertices left, the face
 *    (r'_0, r'_1, r'_2) of the ring in its current order closes the loop when n.N > 0.  A loop with no allowed ear left
 *    stays open and adds no face.  Fill faces follow the kept input faces, by loop (ascending start vertex), then in
 *    cutting order.
 * 7. (smoothIterations > 0) Taubin steps over the output faces: per iteration a step with f = lambda (0 < lambda <= 1)
 *    from the positions, then one with f = mu (-1 <= mu < 0) from the result: x' = x + f (s / k - x) per component, s
 *    the sum, in ascending id, of the k distinct neighbours' positions (starting from 0).  Vertices on an edge held by
 *    other than two output faces stay fixed.  The neighbours come from the sorted directed edge keys.
 * 8. Outputs: d_outVertices [][3] float (the vertices the output faces use, in ascending input index, rounded to
 *    float), d_outIntensity [] (with d_vertexIntensity, copied), d_outTriangles [][3] (renumbered), each the prefix of
 *    its full list (at most maxOutVertices or maxOutTriangles entries).  info_out [3] (may be NULL): m, s and the
 *    threshold of rule 3 (0 when it is off).  stats_out [19] (may be NULL): input triangles; faces dropped as
 *    degenerate, duplicate, long-edge, non-manifold-edge and small-component; components (after rule 4), components
 *    dropped, non-manifold vertices; loops, loops filled, loops left open, boundary half-edges on no loop, fill faces;
 *    full vertex and triangle counts, vertices and triangles written, status.  Returns the full triangle count, or
 *    CS_E_*.  numTriangles == 0 returns 0 (status 0) and makes no CUDA call.
 * - Determinism: two calls give the same bytes; integer atomics only, each with an order-independent result.
 * - Launches (cs_launch_count): validate (only that one when the input is invalid), init, 3 for rule 2, edge keys, 4 for
 *   rule 3, 2 for rule 4, 3 for the links, roots and counts, 1 for rule 5's drop, 6 + R for rule 6 (boundary, count,
 *   write, successors, R = ceil(log2(3 numTriangles + 1)) jumps, loops, ears) plus its copy of the fill faces, 2 for
 *   the kept faces, 2 + 2 smoothIterations for rule 7 and 4 for the output; each stage's only when it is on.  Plus
 *   cub's sorts and scans (not counted).  The host synchronises after the input check, before smoothing when it is on,
 *   and at the end; *ms (may be NULL) gets the event time of the whole call.
 * - Scratch, allocated on the call's stream and freed before it returns: 292 bytes per triangle and 97 per vertex, and
 *   with smoothing 96 more per output triangle, plus cub's storage.
 * - CS_E_ARG, before any CUDA call, naming the argument: numTriangles outside [0, 2^26], removeDegenerate or
 *   removeNonManifold not 0 or 1, longEdgeFactor not finite or < 0, minComponentFaces < 0, minComponentFraction outside
 *   [0, 1], maxHoleEdges not 0 and outside [3, 256], smoothIterations outside [0, 1000], lambda outside (0, 1], mu
 *   outside [-1, 0); then cs_simplify_mesh's checks of numVertices, the buffers and their overlap. */
int cs_clean_mesh(const float *d_vertices, const float *d_vertexIntensity, int numVertices, const int *d_triangles,
                  int numTriangles, int removeDegenerate, double longEdgeFactor, int removeNonManifold,
                  int minComponentFaces, double minComponentFraction, int maxHoleEdges, int smoothIterations,
                  double lambda, double mu, float *d_outVertices, float *d_outIntensity, int maxOutVertices,
                  int *d_outTriangles, int maxOutTriangles, double info_out[3], long long stats_out[19], double *ms);

/* Mesh texturing (Waechter, Moehrle & Goesele, "Let There Be Color!", ECCV 2014, without global seam levelling): for
 * every face one image to take its texture from, the charts of adjacent faces with the same image, and one atlas of
 * the charts' image rectangles with per-corner texture coordinates.  Images and cameras are the dense calls' (pinhole:
 * images with distortion go through cs_undistort_images first); the mesh is in the layout cs_poisson_mesh and
 * cs_simplify_mesh write, device buffers passed in place: d_vertices [numVertices][3] float, d_triangles
 * [numTriangles][3] int32.  All arithmetic below is float64, each operation rounded once in the order written (no
 * contraction); the rules depend on values alone, so two calls give the same bytes.
 * 1. Input and adjacency: status 2 and nothing written when a triangle index lies outside [0, numVertices), a triangle
 *    repeats a vertex, or a vertex some triangle uses has a non-finite coordinate (cs_simplify_mesh's rule 1).  Corner
 *    3t + k starts the edge from corner k to corner k + 1 mod 3.  Two faces are adjacent across an undirected edge when
 *    exactly two faces hold it (found by a radix sort of the keys (min << 32) | max of the corners' edges); an edge with
 *    one face or with three or more gives no adjacency, so a face has at most 3 neighbours.
 * 2. Depth buffers: image a maps a vertex X (float, as float64) to Y = R_a X + t_a, component i
 *    ((R_i0 X_0 + R_i1 X_1) + R_i2 X_2) + t_i, and (u, v) = (((K_0 Y_0 + K_1 Y_1) + K_2 Y_2) / Y_2,
 *    ((K_3 Y_0 + K_4 Y_1) + K_5 Y_2) / Y_2); pixel (x, y) has its centre at integer (x, y).  Every face whose three
 *    vertices have Y_z > 0 is rasterised, front-facing or not, so back faces of open meshes occlude.  With the doubled
 *    area A = (u_1 - u_0)(v_2 - v_0) - (v_1 - v_0)(u_2 - u_0) (corners in face order; A = 0 or not finite: no pixel) and
 *    s = sign(A): edge k from vertex P to vertex Q, P the corner of the lower vertex index, has
 *    e_k = (u_Q - u_P)(y - v_P) - (v_Q - v_P)(x - u_P), and w_k = s e_k, negated when corner k holds the higher index,
 *    so the two faces of an edge see exactly opposite values and no pixel centre on a shared edge is missed.  A pixel in
 *    [0, W - 1] x [0, H - 1] is covered when w_0, w_1, w_2 >= 0 and S = (w_0 + w_1) + w_2 > 0; its depth is
 *    float(1 / (((w_1 / z_0 + w_2 / z_1) + w_0 / z_2) / S)) (perspective-correct, rounded to float once).  The pixel's
 *    key (float bits << 32) | face is combined by 64-bit atomicMin (empty: all ones), so the nearest surface wins, ties
 *    go to the lower face, and the order of execution does not matter.  Images are processed in groups of consecutive
 *    images whose buffers (8 bytes per pixel) fit 1 GiB (at least one image each); the result does not depend on the
 *    grouping.
 * 3. Candidates: with n_f = (p_1 - p_0) x (p_2 - p_0) (cs_simplify_mesh's products), the centroid
 *    c = ((p_0 + p_1) + p_2) / 3, C_a = -R_a^T t_a (component i -((R_0i t_0 + R_1i t_1) + R_2i t_2)) and d = C_a - c,
 *    image a is a candidate of face f when n_f . d > 0; n_f . d >= cos(maxViewAngleDeg pi / 180) (sqrt(n.n) sqrt(d.d))
 *    (the cosine by the host's libm); p_0, p_1, p_2 and c project with Y_z > 0 into [0, W - 1] x [0, H - 1]; at each
 *    of those 4 points the buffer at pixel (floor(u + 0.5), floor(v + 0.5)) is empty, holds f, or has a depth d with
 *    Y_z <= d (1 + depthTol); and the quality q(f, a) = 0.5 |A| (the projected area in pixels) is > 0.  A face keeps
 *    its best 8 candidates by (q descending, image ascending), a set that does not depend on the groups.  A face
 *    without a candidate is unseen: label -1, NaN texture coordinates, in no chart.
 * 4. Labelling: D(f, a) = 1 - q(f, a) / q(f, best), E = sum_f e_f with e_f = D(f, l_f) + lambda times the number of
 *    f's edges whose neighbour g > f is labelled with l_g != l_f (each adjacent pair counted once per shared edge).
 *    Every seen face starts at its best candidate.  The face graph is coloured by Jones-Plassmann with the priority
 *    s(f) = m ^ (m >> 16), m = f 0x9E3779B1 mod 2^32 (cs_simplify_mesh's bijection): in a round, which reads the state
 *    at its start, an uncoloured face whose priority is above every uncoloured neighbour's takes the smallest colour
 *    no coloured neighbour holds (unseen faces take part; at most 4 colours).  A sweep updates the faces of colour 0,
 *    then 1, and so on (ICM, iterated conditional modes: a seen face takes the candidate of lowest local energy
 *    D(f, a) + lambda #{labelled neighbours across an edge with a label != a}, keeping its label on ties, then
 *    preferring the earlier rank).  The call stops after a sweep that changes nothing (status 0) or after maxSweeps
 *    sweeps (status 3).  E never increases; info_out [2] (may be NULL) gets E before and after the sweeps, each summed
 *    in coop.cuh's three-level order (tiles of 2048 faces, groups of 256 tiles, the group partials).
 * 5. Charts: the connected components of adjacent seen faces with equal labels (union-find, each link from the higher
 *    root to the lower, so every root is the lowest face of its chart), ordered by that face.  A chart's rectangle in
 *    its image is x0 = max(0, min floor(u) - padding), x1 = min(W - 1, max ceil(u) + padding) over its faces' corners,
 *    likewise y0, y1 (integer atomics on floor and ceil).
 * 6. Atlas, packed on the host over one copy of the chart table: the charts sorted by (height descending, width
 *    descending, index ascending) go into shelves left to right, a new shelf starting under the current one when the
 *    next chart does not fit in atlasWidth texels; the full atlas height is the sum of the shelf heights, and chart c
 *    lies at (ox, oy).  Its texel (X, Y) is an exact copy of image_a(x0 + X - ox, y0 + Y - oy) (one texel per pixel:
 *    no resampling, and the padding is real image data for bilinear filtering and mipmaps); texels outside every
 *    chart are 0.  A corner's coordinate is (float((u - x0) + ox), float((v - y0) + oy)) in atlas pixels.
 * - Outputs: d_atlas [maxAtlasRows][atlasWidth] float (the prefix of the full atlas's rows); d_uv [numTriangles][3][2]
 *   float, d_faceView [numTriangles] int32 (the label) and d_faceChart [numTriangles] (may be NULL; -1 when unseen),
 *   which always refer to the full atlas; charts_out [maxCharts][8] (host int32) {image, x0, y0, width, height, ox, oy,
 *   faces}, the prefix of the chart list.  stats_out [11] (may be NULL): faces, unseen faces, candidate pairs (before
 *   the cap of 8), colours, Jones-Plassmann rounds, sweeps, labels changed, charts, atlas rows (full), atlas rows
 *   written, status.  Returns the full chart count, or CS_E_*.  numTriangles == 0 returns 0 (stats and info zero) and
 *   makes no CUDA call.
 * - Launches (cs_launch_count): 14 + 2 G + rounds + colours x sweeps for G image groups (validate; edge keys,
 *   adjacency; per group raster and candidates; label start; one per colouring round; two per energy total; per sweep
 *   one per colour; union, roots, chart start, rectangles; texture coordinates, texel copy), 1 when the input is
 *   invalid; plus cub's sort and scan (not counted).  The host reads a few words after the input check, each group,
 *   each colouring round, each total and each sweep, and the chart table (one synchronise each); *ms (may be NULL)
 *   gets the event time of the whole call.
 * - Scratch, allocated on the call's stream and freed before it returns: 272 bytes per face (edge keys and corners and
 *   their sorted copies, neighbours, 8 candidates, labels, two colour arrays, parents, root flags, chart indices, chart
 *   rectangles, the chart table and texel starts), 8 per group of 2048 faces, 8 bytes per pixel of the largest image
 *   group (at most 1 GiB unless one image is larger), 224 per image, plus cub's storage.
 * - CS_E_ARG, before any CUDA call, naming the argument: the dense calls' image and camera checks; numVertices outside
 *   [0, 2^30], numTriangles outside [0, 2^29]; lambda not finite or < 0; maxViewAngleDeg not in (0, 90]; depthTol not
 *   in [0, 1]; padding outside [0, 16]; atlasWidth outside [the largest image width, 32768]; maxSweeps outside
 *   [0, 1000]; maxAtlasRows or maxCharts < 0; NULL or not 4-byte aligned d_vertices with numVertices > 0, d_triangles,
 *   d_uv or d_faceView with numTriangles > 0, d_atlas with maxAtlasRows > 0; a misaligned d_faceChart; NULL charts_out
 *   with maxCharts > 0; and an output (d_atlas, d_uv, d_faceView, d_faceChart) that overlaps another output, the mesh
 *   or an image (one sweep over sorted ranges). */
int cs_texture_mesh(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
                    const float *d_vertices, int numVertices, const int *d_triangles, int numTriangles, double lambda,
                    double maxViewAngleDeg, double depthTol, int padding, int atlasWidth, int maxSweeps,
                    float *d_atlas, int maxAtlasRows, float *d_uv, int *d_faceView, int *d_faceChart,
                    int *charts_out, int maxCharts, double info_out[2], long long stats_out[11], double *ms);

/* Mesh texturing with Waechter, Moehrle & Goesele's view selection (ECCV 2014, section 4.1): cs_texture_mesh with a
 * data term that prefers sharp views, the gradient magnitude integrated over the face's projection (GMI), and the
 * rejection of views whose colour over the face disagrees with the others' (a pedestrian, a car, a reflection seen
 * in one view only).  The arguments are cs_texture_mesh's, with dataTerm, outlierK and outlierMinSigma after
 * numTriangles.  Rules 1, 2 and 4 to 6 are cs_texture_mesh's; rule 3 is replaced by 3a to 3c.  All arithmetic is
 * float64, each operation rounded once in the order written (no contraction); the result depends on values alone,
 * not on scheduling or on the image groups, so two calls give the same bytes.
 * 3a. Samples: a pair (f, a) that passes every test of cs_texture_mesh's rule 3 is sampled over its box, rule 2's
 *    clipped bounding box xlo..xhi, ylo..yhi of f's projection in image a.  Its samples are the box pixels whose
 *    depth-buffer key names f, exactly the pixels where f is visible.  With the box index i = (y - ylo) boxWidth +
 *    (x - xlo), lane j of a warp sums the samples with i = j mod 32 in ascending i (a count n, sum G and sum I), and the
 *    three sums are combined by the xor butterfly 16, 8, 4, 2, 1 (lane 0's value is used).  I is the pixel value (pitch
 *    respected); G is the Sobel magnitude with indices clamped to the image:
 *    gx = ((I(x+1,y-1) - I(x-1,y-1)) + 2 (I(x+1,y) - I(x-1,y))) + (I(x+1,y+1) - I(x-1,y+1)),
 *    gy = ((I(x-1,y+1) - I(x-1,y-1)) + 2 (I(x,y+1) - I(x,y-1))) + (I(x+1,y+1) - I(x+1,y-1)),
 *    G = sqrt(gx gx + gy gy) / 8 (a ramp of slope s gives s).  The means are g = sum G / n and mu = sum I / n; with
 *    n = 0 (a face smaller than a pixel, or hidden at every pixel centre) g and mu are read at the centroid pixel
 *    (floor(uc + 0.5), floor(vc + 0.5)) that rule 3 tested.
 * 3b. Data term: dataTerm 0 is the area, q = 0.5 |A| as in cs_texture_mesh; dataTerm 1 is GMI, q = (0.5 |A|) (g + 1).
 *    The 1 is a floor in grey levels per pixel, so textureless faces still rank by area and never get q = 0; like the
 *    stereo variance floor it assumes images on a 0..255 scale.  A face keeps its best 8 candidates by (q descending,
 *    image ascending), and mu travels with each kept candidate.
 * 3c. Outliers, after every image group and before the labelling: with outlierK > 0, a face with m >= 3 kept
 *    candidates is tested.  med is the median of its m values of mu ((a + b) * 0.5 of the two middle values for even
 *    m), MAD the median of |mu_i - med| likewise, and s = max(1.4826 MAD, outlierMinSigma).  A candidate leaves the
 *    list when |mu_i - med| > outlierK s; the survivors keep their order.  With outlierK >= 1 at least ceil(m / 2)
 *    candidates survive (half the values lie within MAD of med), so a tested face is never left unseen.  When the best
 *    candidate leaves, the face starts at the new first candidate and D (rule 4) is normalised by its q.
 * - Outputs: cs_texture_mesh's.  stats_out [16] (may be NULL): cs_texture_mesh's 11 entries in place (status at
 *   [10]), then samples summed over every passing pair, pairs that fell back to the centroid pixel, faces tested,
 *   candidates removed, and faces whose best candidate was removed.  numTriangles == 0 returns 0 (stats and info
 *   zero) and makes no CUDA call.
 * - Launches (cs_launch_count): 15 + 2 G + rounds + colours x sweeps (the candidate kernel replaced by the sampling
 *   kernel, a warp per face, and one outlier kernel, a thread per face, that always runs), 1 when the input is
 *   invalid.  With dataTerm 0 and outlierK 0 every output and stats_out [0..10] equal cs_texture_mesh's.
 * - Scratch: cs_texture_mesh's plus 64 bytes per face (mu of the 8 candidates) and 32 bytes.
 * - CS_E_ARG, before any CUDA call, naming the argument: cs_texture_mesh's checks; dataTerm not 0 or 1; outlierK not 0
 *   and not in [1, 100] (NaN rejected); outlierMinSigma not finite or not in (0, 1000]. */
int cs_texture_mesh_photo(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
                          const float *d_vertices, int numVertices, const int *d_triangles, int numTriangles,
                          int dataTerm, double outlierK, double outlierMinSigma, double lambda,
                          double maxViewAngleDeg, double depthTol, int padding, int atlasWidth, int maxSweeps,
                          float *d_atlas, int maxAtlasRows, float *d_uv, int *d_faceView, int *d_faceChart,
                          int *charts_out, int maxCharts, double info_out[2], long long stats_out[16], double *ms);

/* Mesh texturing with Waechter, Moehrle & Goesele's view selection and their MRF solved by loopy belief propagation
 * (min-sum) before the ICM sweeps: cs_texture_mesh_photo with rule 4 split into 4a and 4b.  ICM alone stops at the
 * first labelling no single face can improve, so it keeps islands of faces that all prefer another view by a small
 * margin (m faces with D = delta inside a region of another label cost m delta to flip and save 2 lambda); BP passes
 * evidence along the mesh and removes them, which means fewer seams and fewer charts.  The arguments are
 * cs_texture_mesh_photo's, with maxBpSweeps after outlierMinSigma.  Rules 1 to 3c, 5 and 6 are the photo call's.
 * D(f, r) = 1 - q(f, r) / q(f, 0) over f's candidates a_f[0..m_f - 1] (rank r), lambda and E are rule 4's; all arithmetic
 * is float64, each operation rounded once in the order written, and every minimum is exact, so the result depends on
 * values alone, not on scheduling or on the image groups.
 * 4a. Start and colouring: as rule 4; E_0 is E of the start labelling.
 * 4b. Factors: each edge shared by two seen faces is a Potts factor lambda [l_f != l_g] (rule 1's adjacency slots; a
 *    pair that shares two edges has two factors).  Messages: for seen f and slot k (f's edge from corner k to k + 1)
 *    with seen g across it, the message is a vector over g's ranks r', stored at g's slot k', the slot of g whose two
 *    vertex ids are those of f's slot k.  Every message starts at 0.  h(r) = D(f, r) + the messages into f at the slots
 *    j != k, added in ascending j (a fresh sum, never a subtraction from the full sum); M(r') = min(h(r_a) if a_g[r']
 *    is f's candidate at rank r_a else +inf, min_r h(r) + lambda); the message is M(r') - min_r' M(r') (its smallest
 *    entry exactly 0, every entry at most lambda).  Schedule: a sweep takes colours 0, 1, ... in order; a step writes
 *    every message out of every seen face of its colour and reads only messages into faces of that colour, which no
 *    face of the colour writes, so a step is race-free and equals a sequential pass.  Decode, after every sweep:
 *    b_f(r) = D(f, r) + every message into f, added in ascending slot order; the label is a_f[r*], r* the lowest rank of
 *    minimum b.  Keep: E of the decoded labels (rule 4's total) is compared with the kept labelling's; a labelling is
 *    kept when its E is strictly lower.  The start labelling (E_0, sweep 0) is kept first; it is the decode with every
 *    message 0.  Stop: after a sweep in which no message entry changed a bit, or after maxBpSweeps sweeps.  The labels
 *    then become the kept labelling, and rule 4's ICM sweeps run from it unchanged (maxSweeps, status 0 or 3), so
 *    E_final <= E_kept <= E_0.  On a face graph without cycles (a strip) the messages are exact min-marginals after
 *    enough sweeps, and the kept labelling is a minimum of E.
 * - Outputs: cs_texture_mesh_photo's.  info_out [3] (may be NULL): E_0, E after the ICM sweeps (the final E), E of the
 *   labelling BP kept.  stats_out [20] (may be NULL): the photo call's 16 in place (status at [10]), then BP sweeps
 *   run, the sweep whose labelling was kept (0: the start labelling), messages changed in the last BP sweep (0:
 *   converged), faces whose kept label differs from the start label.  With maxBpSweeps 0 every output and
 *   stats_out [0..15] equal cs_texture_mesh_photo's, info_out [2] = info_out [0] and stats_out [16..19] are 0.
 *   numTriangles == 0 returns 0 (stats and info zero) and makes no CUDA call.
 * - Launches (cs_launch_count): 15 + 2 G + rounds + colours x sweeps + (colours + 3) x BP sweeps (per BP sweep one
 *   message step per colour, one decode and two for the energy total), 1 when the input is invalid.  The host reads a
 *   few words after each BP sweep (one synchronise each); the kept labels are a device-to-device copy.
 * - Scratch: cs_texture_mesh_photo's plus 196 bytes per face (the messages [T][3][8] float64, 192, and the kept labels,
 *   4) and 8 bytes.
 * - CS_E_ARG, before any CUDA call, naming the argument: cs_texture_mesh_photo's checks; maxBpSweeps outside
 *   [0, 1000]. */
int cs_texture_mesh_bp(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
                       const float *d_vertices, int numVertices, const int *d_triangles, int numTriangles,
                       int dataTerm, double outlierK, double outlierMinSigma, int maxBpSweeps, double lambda,
                       double maxViewAngleDeg, double depthTol, int padding, int atlasWidth, int maxSweeps,
                       float *d_atlas, int maxAtlasRows, float *d_uv, int *d_faceView, int *d_faceChart,
                       int *charts_out, int maxCharts, double info_out[3], long long stats_out[20], double *ms);

/* Global seam levelling of a textured mesh (Lempitsky & Ivanov 2007 as Waechter, Moehrle & Goesele 2014 apply it,
 * section 4.2): one additive offset per (vertex, label) pair that evens out the colour steps where charts from
 * different images meet, added to the atlas texel by texel.  The inputs are cs_texture_mesh's outputs as it returns
 * them: the mesh (d_vertices [numVertices][3] float, d_triangles [numTriangles][3] int32), d_faceView [numTriangles]
 * (the label, < 0 unseen), d_uv [numTriangles][3][2] float in atlas pixels, the host chart table charts [numCharts][8]
 * {image, x0, y0, width, height, ox, oy, faces} and d_atlas [atlasRows][atlasWidth] float; padding is the value given to
 * cs_texture_mesh.  No images or cameras are needed: every chart's texels are copies of its image.  All arithmetic
 * below is float64, each operation rounded once in the order written (no contraction).
 * 1. Input: status 2, and only stats_out and a zero info_out written, when cs_texture_mesh's rule 1 fails, a seen
 *    face has a non-finite uv, or a seen face lies in no chart of its own label.  A seen face's chart is the one whose rectangle
 *    [ox, ox + width) x [oy, oy + height) holds (floor(u_0), floor(v_0)) of its corner 0 and whose image is the
 *    face's label (the rectangles do not overlap, so at most one holds it); the host builds a row index of the table
 *    (per atlas row, the charts covering it by ox) and the device searches it.
 * 2. Unknowns: one offset g(v, l) per distinct (vertex, label) over the corners of seen faces, in ascending (v, l).
 * 3. Seam edges: an undirected edge held by exactly two faces (cs_texture_mesh's adjacency), both seen, with labels
 *    a < b, endpoints P < Q (vertex ids).  On each side the uv runs from its corner at P to its corner at Q:
 *    x(t) = u_P + t (u_Q - u_P) (likewise y), L_s = sqrt(du^2 + dv^2); S = max(1, ceil(max(L_a, L_b))) samples at
 *    t_k = (k + 0.5) / S.  A side's value I is the bilinear read of the atlas at x(t), y(t): x0 = floor(x), fx = x - x0,
 *    taps x0 and x0 + 1 clamped to that face's chart rectangle (likewise y), r0 = (1 - fx) A(ya, xa) + fx A(ya, xb),
 *    r1 = (1 - fx) A(yb, xa) + fx A(yb, xb), I = (1 - fy) r0 + fy r1.  Sample k counts towards P with w = 1 - t_k and
 *    towards Q with w = t_k: each end of an edge keeps (sum w I_a, sum w I_b, sum w) over its samples in k order.  For
 *    every (v, a, b) the ends at v of the seam edges between a and b are added in sorted edge-key order, and
 *    F(v, a) = (sum w I_a) / (sum w), F(v, b) likewise; the triple gives one seam row
 *    g(v, a) - g(v, b) = F(v, b) - F(v, a) with weight 1.  Seam rows are ordered by (g(v, a), g(v, b)).
 * 4. Smoothness: every distinct (label, min(v, w), max(v, w)) over the edges of seen faces gives g(v, l) - g(w, l) = 0
 *    with weight smoothness; these rows follow the seam rows, ordered by their two unknowns.
 * 5. System: (L_w + regularization I) g = b, L_w the weighted graph Laplacian of the rows (row r: g_i - g_j = d_r with
 *    weight w_r adds w_r to the diagonal of i and j, -w_r off the diagonal, w_r d_r to b_i and -w_r d_r to b_j).
 *    regularization > 0 makes the system symmetric positive definite.
 * 6. Solve: Jacobi-preconditioned CG from g = 0 in float64 in one cooperative kernel; an unknown's incidences are
 *    sorted by a stable radix sort and summed in coop.cuh's piece order, every dot product in its three-level order.
 *    It stops when r.r <= tol^2 b.b (status 0) or after maxIterations (status 3).  Status 1: no seam row; the offsets
 *    are 0 and the atlas is copied bit for bit.
 * 7. Texels: every seen face visits the texels (X, Y) of its chart rectangle inside
 *    [floor(min u) - (padding + 1), ceil(max u) + padding + 1] x (likewise v), each texel centre at integer (X, Y).
 *    Its distance to the face's uv triangle is 0 inside (doubled area A != 0 and w_0, w_1, w_2 >= 0 with
 *    S = (w_0 + w_1) + w_2 > 0 by cs_texture_mesh's lower-vertex edge rule, so shared edges leave no gap; weights
 *    (w_1, w_2, w_0) / S), else the nearest of the three segments k -> k + 1 (t = clamp(((p - a).(b - a)) / |b - a|^2,
 *    0, 1), 0 when |b - a| = 0; ties to the lower k; weights 1 - t, t).  The texel takes the 64-bit atomicMin of
 *    (float(distance) bits << 32) | face.  A texel with a key becomes atlas + float((b_0 o_0 + b_1 o_1) + b_2 o_2), the
 *    winning face's weights at the closest point and its float corner offsets o (d_cornerOffset), the sum in float;
 *    every other texel, and every texel outside every chart, is copied.
 * - Outputs: d_outAtlas [atlasRows][atlasWidth] (a separate buffer); d_cornerOffset [numTriangles][3] float, the
 *   offset g at each corner of a seen face, NaN for an unseen face.  info_out [3] (may be NULL): the seam energy
 *   sum over seam rows of ((F_a + g_a) - (F_b + g_b))^2 before (g = 0) and after, and the true relative residual
 *   sqrt(|b - A g|^2 / |b|^2) (0 when b = 0), each total in coop.cuh's three-level order.  stats_out [8] (may be NULL):
 *   seen faces, unknowns, seam edges, seam rows, smoothness rows, CG iterations, texels visited, status.  Returns the
 *   unknown count, or CS_E_*.  numTriangles == 0: the atlas is copied, status 1.
 * - Determinism: no floating-point atomics; two calls give the same bytes.
 * - Launches (cs_launch_count): 13 whatever the data (validate, chart check; keys, adjacency, unknowns, smoothness
 *   keys, smoothness heads; samples, row heads, rows; one cooperative solve kernel; texel keys, texels), 2 when the
 *   input is invalid; plus cub's sorts and scans (not counted).  The host reads a few words after the input check,
 *   the counts and the seam rows, and after the texels (one synchronise each); *ms (may be NULL) gets the event time
 *   of the whole call.
 * - Scratch, allocated on the call's stream and freed before it returns: 1061 bytes per face (edge, unknown and
 *   smoothness keys and their corners, flags and scans, seam ends, rows, incidences, the CG vectors, an unknown's
 *   range and pieces for up to 3 unknowns per face), 8 bytes per atlas texel (the texel keys), 4 per atlas row and
 *   32 per chart plus 4 per chart row (the table and its row index), plus cub's storage.
 * - CS_E_ARG, before any CUDA call, naming the argument: numVertices outside [0, 2^30], numTriangles outside
 *   [0, 2^29], atlasRows outside [0, 32768], atlasWidth outside [1, 32768], padding outside [0, 16], smoothness not
 *   finite or < 0, regularization not finite or <= 0, maxIterations outside [0, 100000], tol not in [0, 1),
 *   numCharts < 0, NULL charts with numCharts > 0, a chart with an image < 0 or a rectangle outside the atlas, two
 *   charts whose rectangles share a texel (one sweep over x, naming both charts); NULL or
 *   not 4-byte aligned d_vertices with numVertices > 0, d_triangles, d_faceView, d_uv or d_cornerOffset with
 *   numTriangles > 0, d_atlas or d_outAtlas with atlasRows > 0; and an output (d_outAtlas, d_cornerOffset) that
 *   overlaps another output or an input (one sweep over sorted ranges). */
int cs_level_texture_seams(const float *d_vertices, int numVertices, const int *d_triangles, int numTriangles,
                           const int *d_faceView, const float *d_uv, const int *charts, int numCharts,
                           const float *d_atlas, int atlasRows, int atlasWidth, int padding, double smoothness,
                           double regularization, int maxIterations, double tol, float *d_outAtlas,
                           float *d_cornerOffset, double info_out[3], long long stats_out[8], double *ms);

/* Local seam levelling of a textured mesh (Waechter, Moehrle & Goesele 2014, section 4.2, after Perez et al. 2003):
 * Poisson editing of the texel strips along every seam, which removes the steps the global call's per-vertex offsets
 * cannot (a mismatch that varies faster than the mesh or along one seam edge).  The inputs are
 * cs_level_texture_seams's, and d_atlas is normally its output.  All arithmetic below is float64, each operation
 * rounded once in the order written (no contraction).
 * 1. Input: cs_level_texture_seams's rule 1 unchanged (the same checks, status 2, the chart of each seen face).
 * 2. Domain: the texels that cs_level_texture_seams's rule 7 gives a key (every texel of a seen face's chart rectangle
 *    inside its uv box grown by padding + 1); a texel belongs to its key face's chart.  Two texels are neighbours when
 *    they are 4-adjacent, both in the domain and in the same chart, taken in the order (x - 1, y), (x + 1, y),
 *    (x, y - 1), (x, y + 1).
 * 3. Seam texels: cs_level_texture_seams's rule 3 seam edges (sorted by key), sides, sample count S, positions t_k and
 *    bilinear reads I_a, I_b of d_atlas.  Sample k has the target m_k = 0.5 (I_a + I_b) and lands on each side s at
 *    the nearest texel (floor(x + 0.5), floor(y + 0.5)) of x(t_k), y(t_k), clamped to that face's chart rectangle
 *    (always in the domain: within sqrt(2)/2 of the face).  A seam texel's value f* is the sum of the targets landing
 *    on it in (seam edge, side, k) order divided by their count.
 * 4. Strip: the hop distance d is 0 at seam texels and grows by one per neighbour step, computed by stripWidth
 *    synchronous rounds d <- min(d, d of a neighbour + 1).  Free texels have 1 <= d <= stripWidth and are the
 *    unknowns, numbered in row-major atlas order; every other domain texel is fixed.
 * 5. System: for the correction delta = f - g (g the input atlas), with the atlas's own gradients as guidance:
 *    diag_p = the number of neighbours of p, (A delta)_p = diag_p delta_p - sum over free neighbours q of delta_q
 *    (in neighbour order), b_p = sum over seam neighbours q of (f*_q - g_q) (in neighbour order).  Fixed neighbours
 *    hold delta = 0 and a missing neighbour is a Neumann edge.  Every free texel reaches a seam texel through free
 *    texels of decreasing d, so A is irreducibly diagonally dominant, hence symmetric positive definite.
 * 6. Solve: Jacobi-preconditioned CG from delta = 0 in one cooperative kernel, every dot product in coop.cuh's
 *    three-level order; it stops when r.r <= tol^2 b.b (status 0; 0 iterations when b = 0) or after maxIterations
 *    (status 3).  Status 1: no seam texel; the atlas is copied bit for bit.
 * 7. Output, texel by texel: a seam texel becomes float(f*), a free texel float(g + delta), every other texel (fixed,
 *    outside the domain or outside every chart) is copied bit for bit.  Padding texels beyond a seam line are free
 *    texels, so bilinear filtering across the seam reads levelled data.
 * - Outputs: d_outAtlas [atlasRows][atlasWidth] (a separate buffer).  info_out [3] (may be NULL): the sum over seam
 *   texels of (f* - g)^2 in texel order by coop.cuh's three-level order, the true relative residual
 *   sqrt(|b - A delta|^2 / |b|^2) (0 when b = 0), and max |delta| over the free texels.  stats_out [8] (may be NULL):
 *   seen faces, seam edges, samples (sum of S), seam texels, free texels, domain texels, CG iterations, status.
 *   Returns the free-texel count, or CS_E_*.  numTriangles == 0: the atlas is copied, status 1.
 * - Determinism: no floating-point atomics (max |delta| by an integer max of its bits); two calls give the same bytes.
 * - Launches (cs_launch_count): 15 + stripWidth whatever the data (validate, chart check; keys, adjacency, unknowns,
 *   sample counts; texel keys, domain; samples, run heads, seam texels; stripWidth relaxation rounds, free flags;
 *   system; one cooperative solve kernel; output), 2 when the input is invalid; plus cub's sorts and scans (not
 *   counted).  The host reads a few words after the input check, the seam edges, the domain and the strip (one
 *   synchronise each) and after the output; *ms (may be NULL) gets the event time of the whole call.
 * - Scratch, allocated on the call's stream and freed before it returns: 244 bytes per face (edge and unknown keys
 *   and their corners, flags and scans, sample counts), 28 bytes per atlas texel (texel key, chart, two distances,
 *   seam index, free-texel scan), 88 bytes per sample (two slots: texel and target and their sorted copies, run head
 *   and scan, seam texel and f*), 80 bytes per free texel (neighbour codes and the CG vectors) plus 24 per 2048, 4 per
 *   atlas row and 32 per chart plus 4 per chart row, plus cub's storage.
 * - CS_E_ARG, before any CUDA call, naming the argument: cs_level_texture_seams's checks of the mesh, the atlas, the
 *   padding, maxIterations, tol and the chart table (including overlapping rectangles); stripWidth outside [1, 128];
 *   NULL or misaligned buffers as there; and d_outAtlas overlapping an input (one sweep over sorted ranges). */
int cs_level_texture_seams_local(const float *d_vertices, int numVertices, const int *d_triangles, int numTriangles,
                                 const int *d_faceView, const float *d_uv, const int *charts, int numCharts,
                                 const float *d_atlas, int atlasRows, int atlasWidth, int padding, int stripWidth,
                                 int maxIterations, double tol, float *d_outAtlas, double info_out[3],
                                 long long stats_out[8], double *ms);

/* Photometric mesh refinement (Vu, Labatut, Pons & Keriven, PAMI 2012, as OpenMVS's RefineMesh): every free vertex
 * moves so that each ordered image pair (ref, src), reprojected through the mesh, agrees photometrically (windowed
 * NCC), with a thin-plate term that keeps the surface regular.  It recovers the corners, thin parts and fine relief
 * that the Poisson grid and simplification round away.  Images and cameras are the dense calls' (pinhole, images on a
 * 0..255 scale); the mesh is cs_texture_mesh's, d_vertices [numVertices][3] float and d_triangles [numTriangles][3]
 * int32, and the refined vertices go to the separate d_outVertices [numVertices][3]; the topology does not change.
 * pairs [numPairs][2] (host int32) {ref, src}.  All arithmetic is float64, each operation rounded once in the order
 * written (no contraction); no floating-point atomics, so two calls give the same bytes.
 * 1. Input: status 2, with only stats_out and a zero info_out written, when cs_texture_mesh's rule 1 fails.  Every
 *    corner emits the directed edge keys (a << 32) | b and (b << 32) | a of its edge a -> b, sorted; a run of equal
 *    keys is a distinct directed edge and its length is the number of faces holding the edge.  A vertex is fixed when
 *    it starts a run of length != 2 (a boundary or non-manifold edge) or starts no run (no face uses it); every other
 *    vertex is free (F of them) and has its distinct neighbours N(v) in ascending id.  l0 is the mean length of the
 *    distinct undirected edges (the runs with a < b, lengths summed over the sorted positions in coop.cuh's
 *    three-level order).  Fixed vertices never move.
 * 2. Depth buffers: cs_texture_mesh's rule 2, restated in this unit, for every image a pair names, rebuilt at every
 *    evaluation from the vertices being evaluated.
 * 3. Mapping, for pair p = (i, j): pixel x of image i is mapped when its key names a face f and: with rule 2's edge
 *    values w at x, S = (w_0 + w_1) + w_2, screen weights (b_0, b_1, b_2) = (w_1 / S, w_2 / S, w_0 / S), t_k = b_k / z_k
 *    and phi_k = t_k / ((t_0 + t_1) + t_2), the point X = (phi_0 P_0 + phi_1 P_1) + phi_2 P_2 (per component) projects
 *    into j with Y_z > 0 inside [0, W_j - 1] x [0, H_j - 1]; it passes cs_texture_mesh's visibility test in j's buffer
 *    (pixel (floor(u + 0.5), floor(v + 0.5)) empty, naming f, or Y_z <= depth (1 + depthTol)); and n_f . r != 0, with
 *    n_f = (P_1 - P_0) x (P_2 - P_0) and r = X - C_i.  Then J(x) is the bilinear read of j at (u, v): x0 = min(floor(u),
 *    W_j - 2), fx = u - x0 (likewise y0, fy), a = I00 + fx (I10 - I00), b = I01 + fx (I11 - I01), J = a + fy (b - a).
 *    The chain factor is c(x) = (g_u a_u + g_v a_v) / (n_f . r) with the derivatives of that read, g_u = (I10 - I00) +
 *    fy ((I11 - I01) - (I10 - I00)) and g_v = b - a (a change of the proposed design, which read central differences:
 *    this way the gradient is the exact derivative of E inside a cell), and the derivative of j's projection along r,
 *    dY = R_j r (rule 2's row order), a_u = (((K_0 dY_0 + K_1 dY_1) + K_2 dY_2) - u dY_2) / Y_z, a_v likewise with K_3..5
 *    and v.  The scales of n_f and r cancel.
 * 4. Score: x is scored when every pixel of its (2 windowRadius + 1)^2 window lies in image i and is mapped.  Over the
 *    window in row-major order, from 0: sums of I, J, I I, J J and I J; n the window size, mu = sum / n, the raw
 *    variance s = sum sq / n - mu mu, floored as max(s, 1) (the stereo call's floor of 1 grey level^2; J floored when
 *    s < 1); q = sqrt(var_I var_J), NCC = (sum IJ / n - mu_I mu_J) / q, e(x) = 1 - NCC.
 * 5. Image gradient: per scored x, A = 1 / q, B = mu_I A, Cc = NCC / var_J (0 when J is floored), D = Cc mu_J.  For
 *    mapped y, the sums SA, SB, SC, SD over the scored x whose window holds y (x in row-major order, from 0);
 *    dE/dJ(y) = -((((I(y) SA - SB) - J(y) SC) + SD)) / n and s(y) = dE/dJ(y) c(y).
 * 6. Face and vertex gradient: per pair, a warp per face f takes rule 2's clipped box of f in image i and the mapped
 *    box pixels whose key names f; lane l sums s(y) phi_k(y) over the box indices i = l mod 32 in ascending i, the xor
 *    butterfly 16, 8, 4, 2, 1 combines the lanes, and acc_{f,k} = acc_{f,k} + S_{f,k} for every face, pairs in input
 *    order, acc starting at 0 in every evaluation.  The photometric gradient of free v is the sum over its corners
 *    (ascending corner 3f + k) of acc_{f,k} n_f, from 0, each component divided by P0.  P0 is the number of scored
 *    pixels over all pairs at the input mesh: a fixed normaliser, so E does not change scale as coverage changes.
 * 7. Thin plate: for free v, U_v = (the sum of N(v)'s positions in ascending id, from 0) / |N(v)| - V_v;
 *    D_s = F (l0 l0); E_s = (the three-level total over vertices of (U_x U_x + U_y U_y) + U_z U_z, free only) / D_s;
 *    the gradient is (2 / D_s) (-U_v + the sum over free w in N(v), ascending, of U_w / |N(w)|).  E_photo = (the sum over
 *    pairs in input order, from 0, of each pair's three-level total of e over its pixels) / P0, and E = E_photo +
 *    smoothness E_s; G_v = G_photo + smoothness G_s per component.  F = 0 or l0 = 0: E_s and its gradient are 0.
 * 8. Descent: g_rms = sqrt(G2 / F) with G2 the three-level total over free vertices of (G_x G_x + G_y G_y) + G_z G_z
 *    (0 when F = 0).  A step from the accepted vertices with alpha: al = alpha l0, Delta_v = -((al / g_rms) G_v); when
 *    |Delta_v| > 2 al it is scaled by (2 al) / |Delta_v|; the candidate is float(V_v + Delta_v), fixed vertices copied.
 *    The first evaluation is the input (E_0, and P0 from its count).  Status 1: P0 = 0 (the vertices are copied).
 *    Then, before each step: g_rms = 0 or alpha < step / 1024 ends the call with status 0, and maxIterations candidate
 *    evaluations end it with status 3.  alpha starts at step; a candidate whose E is strictly lower than the accepted
 *    E is accepted (with its gradient) and alpha returns to step, otherwise alpha halves.  The output is the accepted
 *    vertices, so E_out <= E_0.  The host decides every branch on totals it reads.
 * - Outputs: d_outVertices.  info_out [4] (may be NULL): E_photo and E_s of the input, then of the output.
 *   stats_out [8] (may be NULL): pairs, free vertices, fixed vertices, P0, evaluations (the first included), accepted
 *   steps, halvings of the final alpha (alpha = step / 2^h), status.  Returns the status, or CS_E_*.  numTriangles == 0:
 *   the vertices are copied, every vertex is fixed and the status is 1, with no kernel launch.
 * - Launches (cs_launch_count): 5 setup kernels (validate; keys; runs; compaction; edge total), then 5 numPairs + 5 per
 *   evaluation (raster of every paired image; per pair map, score, pair total, image gradient, face gather; thin
 *   plate, its total, vertex gradient, its total) and one step kernel before every evaluation but the first: 5 +
 *   evaluations (5 numPairs + 5) + evaluations - 1; 1 when the input is invalid; plus cub's sorts and scan (not
 *   counted).  The host reads a few words after the input check, the setup and each evaluation (one synchronise
 *   each); *ms (may be NULL) gets the event time of the whole call.
 * - Scratch, allocated on the call's stream and freed before it returns: 8 bytes per pixel of every image a pair
 *   names (the depth keys); 50 bytes per pixel of the largest ref image (J, c then s, A, B, Cc, D, the mapped and
 *   scored flags), reused by every pair, and 8 per 2048 of its pixels; 240 bytes per face (directed keys and their
 *   sorted copies, corner keys and corners and their sorted copies, run heads and their scan, the neighbour list, the
 *   corner sums) and 104 per vertex (flags, neighbour and corner ranges, U, two gradients, the candidate), 224 per
 *   paired image and 8 per pair, plus cub's storage.
 * - CS_E_ARG, before any CUDA call, naming the argument: the dense calls' image and camera checks; numVertices outside
 *   [0, 2^30], numTriangles outside [0, 2^28] (the 6 numTriangles directed keys fit an int); numPairs < 0, NULL pairs with numPairs > 0, a pair naming an image
 *   outside [0, numImages) or with ref == src; windowRadius outside [1, 5]; smoothness not finite or < 0; step not in
 *   (0, 1]; maxIterations outside [0, 1000]; depthTol not in [0, 1]; NULL or not 4-byte aligned d_vertices or
 *   d_outVertices with numVertices > 0, d_triangles with numTriangles > 0; and d_outVertices overlapping the mesh or
 *   an image (one sweep over sorted ranges). */
int cs_mesh_refine(const cs_image *images, int numImages, const double *Ks, const double *Rs, const double *ts,
                   const float *d_vertices, int numVertices, const int *d_triangles, int numTriangles,
                   const int *pairs, int numPairs, int windowRadius, double smoothness, double step,
                   int maxIterations, double depthTol, float *d_outVertices, double info_out[4],
                   long long stats_out[8], double *ms);

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
/* The same for cs_verify_essential: h_models[10*numLoops][9] receives every slot's E = (T2 K2)^T Fn (T1 K1) at unit
 * Frobenius norm with its largest-magnitude entry positive (NaN-filled when empty), h_counts[10*numLoops] and h_norm
 * as above. */
int cs_verify_essential_models(const void *d_s1, int n1, const void *d_s2, int n2, const int *d_pairs, int numPairs,
                               const double K1[9], const double K2[9], int numLoops, float thresh,
                               unsigned long long seed, double *h_models, int *h_counts, double h_norm[5]);
/* The steps of cs_absolute_pose_batch up to scoring for one job, with its argument checks (K the job's intrinsics):
 * h_R[4*numLoops][9], h_t[4*numLoops][3] receive every slot's pose (NaN-filled when the slot is empty) and
 * h_counts[4*numLoops] every slot's inlier count.  Returns V, the job's number of valid correspondences (0 for n == 0,
 * with no CUDA call and the outputs untouched). */
int cs_absolute_pose_models(const double *d_points, int numPoints, const cs_pose_job *job, const double K[9],
                            int numLoops, double maxError, double *h_R, double *h_t, int *h_counts);

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
