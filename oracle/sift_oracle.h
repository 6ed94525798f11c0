/*
 * sift_oracle.h -- CPU restatement of the CudaSift hot path (TEST INFRASTRUCTURE ONLY).
 *
 * This is the parity oracle for cudasift_b200.  Nothing in the product path may
 * include, link or call it: only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs use it, and only as the checker.
 *
 * Every function restates one stage of the reference (Celebrandil/CudaSift @5bc874a)
 * and cites the reference file:line it follows.  Where the reference's results depend
 * on how nvcc contracted a*b+c into FMAs, the contraction was read off the SASS of the
 * reference (oracle/build_reference.py) and is replayed here with
 * explicit fmaf() calls; build with -ffp-contract=off -mfma.
 *
 * Pinning status (see DESIGN.md "Oracle"): the reference has no CPU implementation and
 * no golden vectors for extraction; the oracle is pinned against outputs of the
 * reference library itself (oracle/_ref/libcudasift_ref.so) run on the GPU box, stored
 * as fixtures under tests/golden/ by tests/golden/make_golden.py.
 */
#ifndef SIFT_ORACLE_H
#define SIFT_ORACLE_H

#ifdef __cplusplus
extern "C" {
#endif

/* Same 576-byte record as the reference (cudaSift.h:6-22). */
typedef struct {
  float xpos, ypos, scale, sharpness, edgeness, orientation, score, ambiguity;
  int match;
  float match_xpos, match_ypos, match_error, subsampling;
  float empty[3];
  float data[128];
} OracleSiftPoint;

/* ---- filter taps (host side of the reference) ---- */
/* cudaSiftH.cu:315-324 */
void oracle_scaledown_taps(float variance, float k[5]);
/* cudaSiftH.cu:408-419 */
void oracle_lowpass_taps(float sigma, float k[9]);
/* cudaSiftH.cu:439-458; kernel has 8*12*16 floats, entry [oct*192 + scale*16 + j] */
void oracle_laplace_taps(int numOctaves, float initBlur, float *kernel);

/* ---- image stages ---- */
/* cudaSiftD.cu:1986-2037 (LowPassBlock). src and dst share `pitch` (reference quirk Q5). */
void oracle_lowpass(const float *src, float *dst, int w, int h, int pitch, float sigma);
/* cudaSiftD.cu:84-168 (ScaleDown); dst is (w/2)x(h/2). */
void oracle_scaledown(const float *src, float *dst, int w, int h, int pitch, int newpitch);
/* cudaSiftD.cu:170-190 (ScaleUp); dst is (2w)x(2h). */
void oracle_scaleup(const float *src, float *dst, int w, int h, int pitch, int newpitch);
/* cudaSiftD.cu:1753-1793 (LaplaceMultiMem): 7 DoG planes, plane stride h*pitch. */
void oracle_dog(const float *base, float *dog, int w, int h, int pitch,
                const float *taps /* 8 scales x 16, this octave */);

/* cudaSiftD.cu:1292-1431 (FindPointsMultiNew).  Appends to pts[*count..], returns number
 * of candidates dropped by the reference's 32-per-block cap.  `cap32` != 0 reproduces
 * that cap (reference behaviour); 0 keeps every extremum. */
int oracle_find_points(const float *dog, int w, int h, int pitch, float subsampling,
                       float lowestScale, float thresh, float factor, float edgeLimit,
                       OracleSiftPoint *pts, int *count, int maxPts, int cap32);

/* Texture fetch emulation: linear filter, clamp, unnormalised coords, 1.8 fixed-point
 * weights (cudaSiftH.cu:186-205 sets the texture up). */
float oracle_tex2d(const float *img, int w, int h, int pitch, float x, float y);

/* cudaSiftD.cu:972-1057 (ComputeOrientationsCONST) over pts[first..last); secondary
 * orientations are appended at pts[*count..] (if < maxPts). */
void oracle_orientations(const float *img, int w, int h, int pitch, OracleSiftPoint *pts,
                         int first, int last, int *count, int maxPts);
/* cudaSiftD.cu:308-417 (ExtractSiftDescriptorsCONSTNew) over pts[first..last). */
void oracle_descriptors(const float *img, int w, int h, int pitch, OracleSiftPoint *pts,
                        int first, int last, float subsampling);
/* Votes with angi == 8 (quirk Q22: into angle bin 0 of the next cell) in the last oracle_descriptors call. */
int oracle_last_q22(void);

/* cudaSiftH.cu:72-144 (ExtractSift, scaleUp optional).  img is w*h floats with row
 * stride `pitch`.  Returns numPts as the reference reports it (quirk Q1: the finest
 * octave's secondary orientations are not counted); *total receives the number of
 * records written including those. */
/* Test knobs: switch the cap of 32 extrema per block and scale off / on (default on, as in the reference);
 * number of extrema the cap dropped during the last oracle_extract. */
void oracle_set_cap32(int on);
void oracle_set_cap_limit(int n);   /* tests only: a lower limit makes the cap reachable */
int oracle_last_dropped(void);

int oracle_extract(const float *img, int w, int h, int pitch, int numOctaves,
                   float initBlur, float thresh, float lowestScale, int scaleUp,
                   OracleSiftPoint *pts, int maxPts, int *total);

/* matching.cu:301-397 (FindMaxCorr10) + :1090-1206.  Writes score, ambiguity, match,
 * match_xpos, match_ypos of s1[0..n1).  Only p2 < 32*floor(n2/32) are visited (Q7). */
void oracle_match(OracleSiftPoint *s1, int n1, const OracleSiftPoint *s2, int n2);
/* Same, multi-threaded over rows (results identical; used for CPU baselines). */
void oracle_match_mt(OracleSiftPoint *s1, int n1, const OracleSiftPoint *s2, int n2,
                     int nthreads);

/* matching.cu:1000-1087 (FindHomography, RANSAC with rand()).  Tests all numPts points (the
 * reference also visits up to 15 uninitialised padding entries). */
double oracle_find_homography(const OracleSiftPoint *pts, int numPts, float *homography, int *numMatches,
                              int numLoops, float minScore, float maxAmbiguity, float thresh);

#ifdef __cplusplus
}
#endif
#endif
