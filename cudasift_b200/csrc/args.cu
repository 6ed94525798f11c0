// args.cu -- the argument checks of the C ABI (args.h).  Alignment rules differ between calls and stay with each call;
// every call that takes buffers declares them to one range checker, ArgRanges.
#include "args.h"
#include "common.cuh"

#include <algorithm>
#include <array>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <iterator>
#include <memory>
#include <set>
#include <vector>

namespace cs {

int arg_error(const char *fn, const char *fmt, ...)
{
  char bad[256];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(bad, sizeof bad, fmt, ap);
  va_end(ap);
  set_error("%s: invalid argument (CS_E_ARG): %s", fn, bad);
  return CS_E_ARG;
}

static bool misaligned(const void *p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) != 0; }
static size_t record_bytes(int n) { return n > 0 ? (size_t)n * sizeof(SiftPoint) : 0; }

// The byte ranges of one call: each has a kind (names[kind] is a printf pattern that takes the owner, such as
// "jobs[%d].inliers" or "d_points") and an owner (a table entry, or 0), and is exclusive when it may share no byte with
// any other range (it is written, or must stand alone).
// A single call's ranges (at most 4) stay in `local`, so the per-job checks of a batch allocate nothing; a batch
// call's move to `heap`, sized for the `most` it may add.
struct ArgRanges {
  struct Range {
    uintptr_t lo, hi;
    int kind, owner;
    bool exclusive;
  };
  const char *const *names;
  Range local[4], *rs = local;
  std::unique_ptr<Range[]> heap;
  size_t n = 0, cap = 4;

  ArgRanges(const char *const *names_, size_t most) : names(names_)
  {
    if (most > cap) grow(most);
  }
  void grow(size_t want)
  {
    Range *p = new Range[want];
    std::copy(rs, rs + n, p);
    heap.reset(p);
    rs = p;
    cap = want;
  }
  void add(const void *p, size_t bytes, int kind, int owner, bool exclusive)
  {
    if (!bytes) return;
    if (n == cap) grow(2 * cap);
    const uintptr_t lo = reinterpret_cast<uintptr_t>(p);
    rs[n++] = {lo, lo + bytes, kind, owner, exclusive};
  }
  // The ranges sorted by (start, kind, owner) and swept once (O(n log n)): a range that starts before an earlier one
  // ends overlaps it.  The first conflict found is reported as "<A> and <B> overlap", A the range of the lower
  // (kind, owner).
  int check(const char *fn)
  {
    std::sort(rs, rs + n, [](const Range &a, const Range &b) {
      return a.lo != b.lo ? a.lo < b.lo : a.kind != b.kind ? a.kind < b.kind : a.owner < b.owner;
    });
    const Range *anyEnd = nullptr, *exclEnd = nullptr;   // the earlier ranges (and exclusive ones) that end last
    for (const Range *x_ = rs; x_ != rs + n; x_++) {
      const Range &x = *x_;
      const Range *hit = nullptr;
      if (x.exclusive && anyEnd && anyEnd->hi > x.lo) hit = anyEnd;
      else if (exclEnd && exclEnd->hi > x.lo) hit = exclEnd;
      if (hit) {
        const bool xFirst = x.kind != hit->kind ? x.kind < hit->kind : x.owner < hit->owner;
        const Range &a = xFirst ? x : *hit, &b = xFirst ? *hit : x;
        char na[48], nb[48];
        snprintf(na, sizeof na, names[a.kind], a.owner);
        snprintf(nb, sizeof nb, names[b.kind], b.owner);
        return arg_error(fn, "%s and %s overlap", na, nb);
      }
      if (!anyEnd || x.hi > anyEnd->hi) anyEnd = &x;
      if (x.exclusive && (!exclEnd || x.hi > exclEnd->hi)) exclEnd = &x;
    }
    return 0;
  }
};

int check_sets(const char *fn, const void *s1, int n1, const void *s2, int n2, int mode)
{
  if (n1 < 0 || n2 < 0) return arg_error(fn, "n1 and n2 must be >= 0");
  if ((n1 > 0 && !s1) || (n2 > 0 && !s2)) return arg_error(fn, "a set with records needs a pointer");
  if (mode < 0 || mode > 2) return arg_error(fn, "mode must be 0 (auto), 1 (exact) or 2 (tensor)");
  return 0;
}

// The buffers of a single call: buf[k] of bytes[k] bytes, named names[k], then the records of set 1 and set 2 (named
// names[n] and names[n + 1]).  Every non-empty buffer is 8-byte aligned and shares no byte with another buffer or a
// record range; the record ranges may overlap each other unless the call writes them.
static int call_buffers(const char *fn, const void *s1, int n1, const void *s2, int n2, bool setsWritten,
                        const void *const *buf, const size_t *bytes, const char *const *names, int n)
{
  for (int k = 0; k < n; k++)
    if (bytes[k] && misaligned(buf[k], 8)) return arg_error(fn, "%s must be 8-byte aligned", names[k]);
  ArgRanges rs(names, n + 2);
  for (int k = 0; k < n; k++) rs.add(buf[k], bytes[k], k, 0, true);
  rs.add(s1, record_bytes(n1), n, 0, setsWritten);
  rs.add(s2, record_bytes(n2), n + 1, 0, setsWritten);
  return rs.check(fn);
}

// The pairs buffer of the mutual and ratio matchers: maxPairs int2.
static int check_pairs(const char *fn, const void *s1, int n1, const void *s2, int n2, bool setsWritten,
                       const void *pairs, int maxPairs)
{
  if (maxPairs < 0) return arg_error(fn, "maxPairs must be >= 0");
  if (maxPairs > 0 && !pairs) return arg_error(fn, "maxPairs > 0 needs a pairs buffer");
  static const char *const names[3] = {"pairs", "s1", "s2"};
  const size_t bytes = (size_t)maxPairs * sizeof(int2);
  return call_buffers(fn, s1, n1, s2, n2, setsWritten, &pairs, &bytes, names, 1);
}

int mutual_args(const char *fn, const void *s1, int n1, const void *s2, int n2, const void *pairs, int maxPairs,
                int mode)
{
  const int r = check_sets(fn, s1, n1, s2, n2, mode);
  return r < 0 ? r : check_pairs(fn, s1, n1, s2, n2, true, pairs, maxPairs);
}

int ratio_args(const char *fn, const void *s1, int n1, const void *s2, int n2, float maxRatio, float maxDistance,
               const void *pairs, int maxPairs, int mode)
{
  int r;
  if ((r = check_sets(fn, s1, n1, s2, n2, mode)) < 0) return r;
  if (std::isnan(maxRatio) || std::isnan(maxDistance)) return arg_error(fn, "maxRatio and maxDistance must not be NaN");
  return check_pairs(fn, s1, n1, s2, n2, false, pairs, maxPairs);
}

int verify_args(const char *fn, const void *s1, int n1, const void *s2, int n2, const void *pairs, int numPairs,
                int model, int numLoops, float thresh, const double *model_out, const void *inliers, int maxInliers)
{
  int r;
  if ((r = check_sets(fn, s1, n1, s2, n2, 0)) < 0) return r;              // mode 0: the verifier has one path
  if (numPairs < 0) return arg_error(fn, "numPairs must be >= 0");
  if (numPairs > 0 && !pairs) return arg_error(fn, "numPairs > 0 needs a pairs buffer");
  if (model != CS_GEOM_HOMOGRAPHY && model != CS_GEOM_FUNDAMENTAL)
    return arg_error(fn, "model must be 1 (homography) or 2 (fundamental)");
  if (numLoops < 1 || numLoops > 65536) return arg_error(fn, "numLoops must be in [1, 65536]");
  if (!std::isfinite(thresh) || thresh <= 0.0f) return arg_error(fn, "thresh must be finite and > 0");
  if (!model_out) return arg_error(fn, "model_out must not be NULL");
  if (maxInliers < 0) return arg_error(fn, "maxInliers must be >= 0");
  if (maxInliers > 0 && !inliers) return arg_error(fn, "maxInliers > 0 needs an inliers buffer");
  static const char *const names[4] = {"pairs", "inliers", "s1", "s2"};
  const void *buf[2] = {pairs, inliers};
  const size_t bytes[2] = {(size_t)numPairs * sizeof(int2), (size_t)maxInliers * sizeof(int2)};
  return call_buffers(fn, s1, n1, s2, n2, false, buf, bytes, names, 2);
}

int knn_out_args(const char *fn, const void *s1, int n1, const void *s2, int n2, const int *idx, const float *score)
{
  if (n1 > 0 && (!idx || !score)) return arg_error(fn, "n1 > 0 needs idx and score buffers");
  static const char *const names[4] = {"idx", "score", "s1", "s2"};
  const void *buf[2] = {idx, score};
  const size_t bytes[2] = {(size_t)n1 * 2 * sizeof(int), (size_t)n1 * 2 * sizeof(float)};
  return call_buffers(fn, s1, n1, s2, n2, false, buf, bytes, names, 2);
}

int guided_args(const char *fn, int model, const double *model_in, float thresh)
{
  if (model != CS_GEOM_HOMOGRAPHY && model != CS_GEOM_FUNDAMENTAL)
    return arg_error(fn, "model must be 1 (homography) or 2 (fundamental)");
  if (!model_in) return arg_error(fn, "model_in must not be NULL");
  double s = 0.0;
  for (int k = 0; k < 9; k++) {
    if (!std::isfinite(model_in[k])) return arg_error(fn, "model_in must be finite");
    s += model_in[k] * model_in[k];
  }
  if (!(s > 0.0 && std::isfinite(s))) return arg_error(fn, "model_in must not be all zero (and its norm must be finite)");
  if (!std::isfinite(thresh) || thresh <= 0.0f) return arg_error(fn, "thresh must be finite and > 0");
  return 0;
}

// Intrinsics: a finite row-major pinhole K (skew allowed) with K[3] = K[6] = K[7] = 0, K[8] = 1, K[0] > 0 and K[4] > 0.
static int check_intrinsics(const char *fn, const double *K, const char *name)
{
  bool ok = K != nullptr;
  for (int k = 0; k < 9 && ok; k++) ok = std::isfinite(K[k]);
  if (!ok || K[3] != 0.0 || K[6] != 0.0 || K[7] != 0.0 || K[8] != 1.0 || !(K[0] > 0.0) || !(K[4] > 0.0))
    return arg_error(fn, "%s must be a finite pinhole matrix (K[3] = K[6] = K[7] = 0, K[8] = 1, K[0] > 0, K[4] > 0)",
                     name);
  return 0;
}

int essential_args(const char *fn, const void *s1, int n1, const void *s2, int n2, const void *pairs, int numPairs,
                   const double *K1, const double *K2, int numLoops, float thresh, const double *E, const double *R,
                   const double *t, const void *inliers, int maxInliers)
{
  int r;
  if (!E || !R || !t) return arg_error(fn, "E_out, R_out and t_out must not be NULL");
  if ((r = verify_args(fn, s1, n1, s2, n2, pairs, numPairs, CS_GEOM_FUNDAMENTAL, numLoops, thresh, E, inliers,
                       maxInliers)) < 0)
    return r;
  if ((r = check_intrinsics(fn, K1, "K1")) < 0) return r;
  return check_intrinsics(fn, K2, "K2");
}

// The common arguments, every job's as its single call checks them (named "<fn>: jobs[p]"), the total pair count, then
// the inlier buffers against every other job's buffers and records.
int verify_batch_args(const char *fn, const cs_verify_job *jobs, int numJobs, int model, int numLoops, float thresh,
                      const double *K1s, const double *K2s, bool essential)
{
  int r;
  if (numJobs < 0 || numJobs > 65536) return arg_error(fn, "numJobs must be in [0, 65536]");
  if (numJobs > 0 && !jobs) return arg_error(fn, "numJobs > 0 needs a jobs array");
  if (essential && numJobs > 0 && (!K1s || !K2s)) return arg_error(fn, "K1s and K2s must not be NULL");
  long long total = 0;
  const double dummy = 0.0;
  for (int p = 0; p < numJobs; p++) {
    const cs_verify_job &j = jobs[p];
    char name[96];
    snprintf(name, sizeof name, "%s: jobs[%d]", fn, p);
    if ((r = verify_args(name, j.s1, j.n1, j.s2, j.n2, j.pairs, j.numPairs, model, numLoops, thresh, &dummy, j.inliers,
                         j.maxInliers)) < 0)
      return r;
    if (essential && ((r = check_intrinsics(name, K1s + 9 * (size_t)p, "K1s[p]")) < 0 ||
                      (r = check_intrinsics(name, K2s + 9 * (size_t)p, "K2s[p]")) < 0))
      return r;
    if ((total += j.numPairs) > INT_MAX) return arg_error(fn, "the total numPairs exceeds INT_MAX at jobs[%d]", p);
  }
  // an inlier buffer (written) may overlap no other range; a job's own were checked above
  static const char *const names[4] = {"jobs[%d].inliers", "jobs[%d].pairs", "jobs[%d].s1", "jobs[%d].s2"};
  ArgRanges rs(names, 4 * (size_t)numJobs);
  for (int p = 0; p < numJobs; p++) {
    const cs_verify_job &j = jobs[p];
    rs.add(j.inliers, (size_t)j.maxInliers * sizeof(int2), 0, p, true);
    rs.add(j.pairs, (size_t)j.numPairs * sizeof(int2), 1, p, false);
    rs.add(j.s1, record_bytes(j.n1), 2, p, false);
    rs.add(j.s2, record_bytes(j.n2), 3, p, false);
  }
  return rs.check(fn);
}

// Every set of a cs_match_set table (named sets[s]).
static int check_set_table(const char *fn, const cs_match_set *sets, int numSets)
{
  for (int s = 0; s < numSets; s++) {
    if (sets[s].n < 0) return arg_error(fn, "sets[%d]: n must be >= 0", s);
    if (sets[s].n > 0 && !sets[s].pts) return arg_error(fn, "sets[%d]: a set with records needs a pointer", s);
  }
  return 0;
}

// The common arguments, every set (named sets[s]) and job (jobs[p]), then the pair buffers against each other and
// against every set's records.
int ratio_batch_args(const char *fn, const cs_match_set *sets, int numSets, const cs_match_job *jobs, int numJobs,
                     float maxRatio, float maxDistance, const int *counts_out)
{
  if (numSets < 0 || numSets > 65536) return arg_error(fn, "numSets must be in [0, 65536]");
  if (numJobs < 0 || numJobs > 65536) return arg_error(fn, "numJobs must be in [0, 65536]");
  if (numSets > 0 && !sets) return arg_error(fn, "numSets > 0 needs a sets array");
  if (numJobs > 0 && !jobs) return arg_error(fn, "numJobs > 0 needs a jobs array");
  if (numJobs > 0 && !counts_out) return arg_error(fn, "counts_out must not be NULL");
  if (std::isnan(maxRatio) || std::isnan(maxDistance)) return arg_error(fn, "maxRatio and maxDistance must not be NaN");
  const int r = check_set_table(fn, sets, numSets);
  if (r < 0) return r;
  for (int p = 0; p < numJobs; p++) {
    const cs_match_job &j = jobs[p];
    if (j.set1 < 0 || j.set1 >= numSets || j.set2 < 0 || j.set2 >= numSets)
      return arg_error(fn, "jobs[%d]: set1 and set2 must be in [0, numSets)", p);
    if (j.maxPairs < 0) return arg_error(fn, "jobs[%d]: maxPairs must be >= 0", p);
    if (j.maxPairs > 0 && !j.pairs) return arg_error(fn, "jobs[%d]: maxPairs > 0 needs a pairs buffer", p);
    if (j.maxPairs > 0 && misaligned(j.pairs, 8)) return arg_error(fn, "jobs[%d]: pairs must be 8-byte aligned", p);
  }
  static const char *const names[2] = {"jobs[%d].pairs", "sets[%d].pts"};
  ArgRanges rs(names, (size_t)numSets + numJobs);
  for (int p = 0; p < numJobs; p++) rs.add(jobs[p].pairs, (size_t)jobs[p].maxPairs * sizeof(int2), 0, p, true);
  for (int s = 0; s < numSets; s++) rs.add(sets[s].pts, record_bytes(sets[s].n), 1, s, false);
  return rs.check(fn);
}

// Those of cs_match_ratio_batch, then every job's model as the single call checks it (named jobs[p]).
int guided_batch_args(const char *fn, const cs_match_set *sets, int numSets, const cs_match_job *jobs, int numJobs,
                      const int *models, const double *models_in, float thresh, float maxRatio, float maxDistance,
                      const int *counts_out)
{
  int r;
  if ((r = ratio_batch_args(fn, sets, numSets, jobs, numJobs, maxRatio, maxDistance, counts_out)) < 0) return r;
  if (numJobs > 0 && (!models || !models_in)) return arg_error(fn, "models and models_in must not be NULL");
  for (int p = 0; p < numJobs; p++) {
    char name[96];
    snprintf(name, sizeof name, "%s: jobs[%d]", fn, p);
    if ((r = guided_args(name, models[p], models_in + 9 * (size_t)p, thresh)) < 0) return r;
  }
  return 0;
}

// The counts and tables, every image (imageSizes[a]) and list (lists[p]), the outputs, then the outputs against each
// other and every pair list.
int tracks_args(const char *fn, const int *imageSizes, int numImages, const cs_track_list *lists, int numLists,
                int minLength, const int *trackOf, const int *offsets, int maxTracks, const int *members,
                int maxMembers, int *N, int *P)
{
  if (numImages < 0 || numImages > (1 << 24)) return arg_error(fn, "numImages must be in [0, 2^24]");
  if (numLists < 0 || numLists > (1 << 24)) return arg_error(fn, "numLists must be in [0, 2^24]");
  if (numImages > 0 && !imageSizes) return arg_error(fn, "numImages > 0 needs an imageSizes array");
  if (numLists > 0 && !lists) return arg_error(fn, "numLists > 0 needs a lists array");
  long long n = 0, pairs = 0;
  for (int a = 0; a < numImages; a++) {
    if (imageSizes[a] < 0) return arg_error(fn, "imageSizes[%d] must be >= 0", a);
    if ((n += imageSizes[a]) > INT_MAX) return arg_error(fn, "imageSizes[%d]: the sizes pass INT_MAX", a);
  }
  for (int p = 0; p < numLists; p++) {
    const cs_track_list &l = lists[p];
    if (l.image1 < 0 || l.image1 >= numImages || l.image2 < 0 || l.image2 >= numImages)
      return arg_error(fn, "lists[%d]: image1 and image2 must be in [0, numImages)", p);
    if (l.numPairs < 0) return arg_error(fn, "lists[%d]: numPairs must be >= 0", p);
    if (l.numPairs > 0 && !l.pairs) return arg_error(fn, "lists[%d]: numPairs > 0 needs a pairs buffer", p);
    if (l.numPairs > 0 && misaligned(l.pairs, 8)) return arg_error(fn, "lists[%d]: pairs must be 8-byte aligned", p);
    if ((pairs += l.numPairs) > INT_MAX) return arg_error(fn, "lists[%d]: the pair counts pass INT_MAX", p);
  }
  if (minLength < 2) return arg_error(fn, "minLength must be >= 2");
  if (maxTracks < 0 || maxMembers < 0) return arg_error(fn, "maxTracks and maxMembers must be >= 0");
  if (maxTracks > 0 && !offsets) return arg_error(fn, "maxTracks > 0 needs d_offsets");
  if (maxMembers > 0 && !members) return arg_error(fn, "maxMembers > 0 needs d_members");
  if (misaligned(trackOf, 4) || misaligned(offsets, 4))
    return arg_error(fn, "d_trackOf and d_offsets must be 4-byte aligned");
  if (misaligned(members, 8)) return arg_error(fn, "d_members must be 8-byte aligned");
  // the outputs (written) and the pair lists (read)
  static const char *const names[4] = {"d_trackOf", "d_offsets", "d_members", "lists[%d].pairs"};
  ArgRanges rs(names, (size_t)numLists + 3);
  if (trackOf) rs.add(trackOf, (size_t)n * sizeof(int), 0, 0, true);
  if (offsets) rs.add(offsets, ((size_t)maxTracks + 1) * sizeof(int), 1, 0, true);
  rs.add(members, (size_t)maxMembers * sizeof(int2), 2, 0, true);
  for (int p = 0; p < numLists; p++) rs.add(lists[p].pairs, (size_t)lists[p].numPairs * sizeof(int2), 3, p, false);
  *N = (int)n;
  *P = (int)pairs;
  return rs.check(fn);
}

// The images of cs_triangulate_tracks and cs_bundle_adjust: the counts, every set (sets[a]) and camera (Ks[a], Rs[a],
// ts[a]).
static int camera_args(const char *fn, const cs_match_set *sets, int numImages, const double *Ks, const double *Rs,
                       const double *ts, int numTracks, int numMembers)
{
  if (numImages < 0 || numImages > (1 << 24)) return arg_error(fn, "numImages must be in [0, 2^24]");
  if (numTracks < 0) return arg_error(fn, "numTracks must be >= 0");
  if (numMembers < 0) return arg_error(fn, "numMembers must be >= 0");
  if (numImages > 0 && (!sets || !Ks || !Rs || !ts)) return arg_error(fn, "numImages > 0 needs sets, Ks, Rs and ts");
  int r = check_set_table(fn, sets, numImages);
  if (r < 0) return r;
  for (int a = 0; a < numImages; a++) {
    char name[32];
    snprintf(name, sizeof name, "Ks[%d]", a);
    if ((r = check_intrinsics(fn, Ks + 9 * (size_t)a, name)) < 0) return r;
    const double *R = Rs + 9 * (size_t)a, *t = ts + 3 * (size_t)a;
    bool ok = true;
    for (int k = 0; k < 9; k++) ok = ok && std::isfinite(R[k]);
    for (int i = 0; i < 3 && ok; i++)
      for (int j = 0; j < 3; j++) {
        const double d = R[3 * i] * R[3 * j] + R[3 * i + 1] * R[3 * j + 1] + R[3 * i + 2] * R[3 * j + 2];
        ok = ok && std::fabs(d - (i == j ? 1.0 : 0.0)) <= 1e-6;
      }
    const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) +
                       R[2] * (R[3] * R[7] - R[4] * R[6]);
    if (!ok || !(det > 0.0))
      return arg_error(fn, "Rs[%d] must be a finite rotation (R R^T = I within 1e-6, det R > 0)", a);
    if (!std::isfinite(t[0]) || !std::isfinite(t[1]) || !std::isfinite(t[2]))
      return arg_error(fn, "ts[%d] must be finite", a);
  }
  return 0;
}

// The images (camera_args), the parameters, the buffers, then the outputs against each other, the tracks and every
// set's records.
int triangulate_args(const char *fn, const cs_match_set *sets, int numImages, const double *Ks, const double *Rs,
                     const double *ts, const int *offsets, int numTracks, const int *members, int numMembers,
                     int numTrials, double maxError, double minTriAngle, const double *points, const int *counts,
                     const float *errors, const unsigned char *inlier)
{
  const int r = camera_args(fn, sets, numImages, Ks, Rs, ts, numTracks, numMembers);
  if (r < 0) return r;
  if (numTrials < 1 || numTrials > (1 << 20)) return arg_error(fn, "numTrials must be in [1, 2^20]");
  if (!std::isfinite(maxError) || !(maxError > 0.0)) return arg_error(fn, "maxError must be finite and > 0");
  if (!std::isfinite(minTriAngle) || !(minTriAngle >= 0.0) || !(minTriAngle < 180.0))
    return arg_error(fn, "minTriAngle must be finite and in [0, 180)");
  if (numTracks > 0 && !offsets) return arg_error(fn, "numTracks > 0 needs d_offsets");
  if (numTracks > 0 && (!points || !counts)) return arg_error(fn, "numTracks > 0 needs d_points and d_counts");
  if (numMembers > 0 && !members) return arg_error(fn, "numMembers > 0 needs d_members");
  if (misaligned(offsets, 4) || misaligned(counts, 4) || misaligned(errors, 4))
    return arg_error(fn, "d_offsets, d_counts and d_errors must be 4-byte aligned");
  if (misaligned(members, 8) || misaligned(points, 8))
    return arg_error(fn, "d_members and d_points must be 8-byte aligned");
  // the outputs (written), the tracks and the records (read)
  static const char *const names[7] = {"d_points", "d_counts", "d_errors", "d_inlier", "d_offsets", "d_members",
                                       "sets[%d].pts"};
  ArgRanges rs(names, (size_t)numImages + 6);
  if (numTracks > 0) {
    rs.add(points, (size_t)numTracks * 3 * sizeof(double), 0, 0, true);
    rs.add(counts, (size_t)numTracks * sizeof(int), 1, 0, true);
    rs.add(offsets, ((size_t)numTracks + 1) * sizeof(int), 4, 0, false);
  }
  if (errors) rs.add(errors, (size_t)numMembers * sizeof(float), 2, 0, true);
  if (inlier) rs.add(inlier, (size_t)numMembers, 3, 0, true);
  rs.add(members, (size_t)numMembers * sizeof(int2), 5, 0, false);
  for (int a = 0; a < numImages; a++) rs.add(sets[a].pts, record_bytes(sets[a].n), 6, a, false);
  return rs.check(fn);
}

// The images (camera_args), the gauge codes, the parameters, the buffers, then the outputs against each other, the
// tracks, d_use and every set's records.
int bundle_args(const char *fn, const cs_match_set *sets, int numImages, const double *Ks, const double *Rs,
                const double *ts, const unsigned char *fixed, const int *offsets, int numTracks, const int *members,
                int numMembers, const unsigned char *use, const double *points, int maxIterations,
                int maxLinearIterations, double linearTol, double maxError, const double *R_out, const double *t_out,
                const float *errors, const unsigned char *inlier, const double *cost_out)
{
  const int r = camera_args(fn, sets, numImages, Ks, Rs, ts, numTracks, numMembers);
  if (r < 0) return r;
  for (int a = 0; fixed && a < numImages; a++)
    if (fixed[a] > 4) return arg_error(fn, "fixed[%d] must be 0 (free), 1 (held) or 2..4 (t[fixed - 2] held)", a);
  if (maxIterations < 0 || maxIterations > 1000) return arg_error(fn, "maxIterations must be in [0, 1000]");
  if (maxLinearIterations < 1 || maxLinearIterations > 10000)
    return arg_error(fn, "maxLinearIterations must be in [1, 10000]");
  if (!(linearTol > 0.0) || !(linearTol < 1.0)) return arg_error(fn, "linearTol must be in (0, 1)");
  if (!std::isfinite(maxError) || !(maxError > 0.0)) return arg_error(fn, "maxError must be finite and > 0");
  if (numImages > 0 && (!R_out || !t_out)) return arg_error(fn, "numImages > 0 needs R_out and t_out");
  if (!cost_out) return arg_error(fn, "cost_out must not be NULL");
  if (numTracks > 0 && (!offsets || !points)) return arg_error(fn, "numTracks > 0 needs d_offsets and d_points");
  if (numMembers > 0 && !members) return arg_error(fn, "numMembers > 0 needs d_members");
  if (misaligned(offsets, 4) || misaligned(errors, 4))
    return arg_error(fn, "d_offsets and d_errors must be 4-byte aligned");
  if (misaligned(members, 8) || misaligned(points, 8))
    return arg_error(fn, "d_members and d_points must be 8-byte aligned");
  // the outputs (written), the inputs and the records (read)
  static const char *const names[7] = {"d_points", "d_errors", "d_inlier", "d_offsets", "d_members", "d_use",
                                       "sets[%d].pts"};
  ArgRanges rs(names, (size_t)numImages + 6);
  if (numTracks > 0) {
    rs.add(points, (size_t)numTracks * 3 * sizeof(double), 0, 0, true);
    rs.add(offsets, ((size_t)numTracks + 1) * sizeof(int), 3, 0, false);
  }
  if (errors) rs.add(errors, (size_t)numMembers * sizeof(float), 1, 0, true);
  if (inlier) rs.add(inlier, (size_t)numMembers, 2, 0, true);
  rs.add(members, (size_t)numMembers * sizeof(int2), 4, 0, false);
  if (use) rs.add(use, (size_t)numMembers, 5, 0, false);
  for (int a = 0; a < numImages; a++) rs.add(sets[a].pts, record_bytes(sets[a].n), 6, a, false);
  return rs.check(fn);
}

// The intrinsic arguments of cs_bundle_adjust_intrinsics, then its host arrays: an output may equal its own input
// exactly (K_out == Ks, dist_out == dists, R_out == Rs, t_out == ts); otherwise no output shares a byte with another
// output or with any of the four inputs.
int bundle_intrinsics_args(const char *fn, int numImages, const double *Ks, const double *dists,
                           const unsigned char *refine, int loss, double lossScale, const double *Rs, const double *ts,
                           const double *K_out, const double *dist_out, const double *R_out, const double *t_out)
{
  for (int a = 0; refine && a < numImages; a++)
    if (refine[a] > 7) return arg_error(fn, "refine[%d] must be a mask of bits 0 (focal), 1 (k1) and 2 (k2)", a);
  if (loss < 0 || loss > 2) return arg_error(fn, "loss must be 0 (trivial), 1 (soft-L1) or 2 (Cauchy)");
  if (!std::isfinite(lossScale) || !(lossScale > 0.0)) return arg_error(fn, "lossScale must be finite and > 0");
  for (int a = 0; dists && a < numImages; a++)
    if (!std::isfinite(dists[2 * (size_t)a]) || !std::isfinite(dists[2 * (size_t)a + 1]))
      return arg_error(fn, "dists[%d] must be finite", a);
  if (numImages <= 0) return 0;
  static const char *const names[8] = {"K_out", "dist_out", "R_out", "t_out", "Ks", "dists", "Rs", "ts"};
  const double *outs[4] = {K_out, dist_out, R_out, t_out}, *ins[4] = {Ks, dists, Rs, ts};
  const size_t per[4] = {9, 2, 9, 3};
  ArgRanges rs(names, 8);
  for (int k = 0; k < 4; k++) {
    const size_t bytes = (size_t)numImages * per[k] * sizeof(double);
    if (outs[k]) rs.add(outs[k], bytes, k, 0, true);
    if (ins[k] && ins[k] != outs[k]) rs.add(ins[k], bytes, 4 + k, 0, false);
  }
  return rs.check(fn);
}

// The images, the intrinsics and the outputs of cs_undistort_records: d_out[a] is 4-byte aligned and either is
// sets[a].pts exactly (in place) or shares no byte with another output or any set's records.
int undistort_args(const char *fn, const cs_match_set *sets, int numImages, const double *Ks, const double *dists,
                   void *const *d_out, long long *total)
{
  if (numImages < 0 || numImages > (1 << 24)) return arg_error(fn, "numImages must be in [0, 2^24]");
  if (numImages > 0 && (!sets || !Ks || !d_out)) return arg_error(fn, "numImages > 0 needs sets, Ks and d_out");
  int r = check_set_table(fn, sets, numImages);
  if (r < 0) return r;
  long long n = 0;
  for (int a = 0; a < numImages; a++) {
    char name[32];
    snprintf(name, sizeof name, "Ks[%d]", a);
    if ((r = check_intrinsics(fn, Ks + 9 * (size_t)a, name)) < 0) return r;
    if (dists && (!std::isfinite(dists[2 * (size_t)a]) || !std::isfinite(dists[2 * (size_t)a + 1])))
      return arg_error(fn, "dists[%d] must be finite", a);
    if (sets[a].n > 0 && !d_out[a]) return arg_error(fn, "d_out[%d]: a set with records needs an output", a);
    if (sets[a].n > 0 && misaligned(d_out[a], 4)) return arg_error(fn, "d_out[%d] must be 4-byte aligned", a);
    n += sets[a].n;
  }
  // the outputs (written; an in-place set is its own output) and the records (read)
  static const char *const names[2] = {"d_out[%d]", "sets[%d].pts"};
  ArgRanges rs(names, 2 * (size_t)numImages);
  for (int a = 0; a < numImages; a++) {
    const size_t bytes = record_bytes(sets[a].n);
    rs.add(d_out[a], bytes, 0, a, true);
    if (d_out[a] != sets[a].pts) rs.add(sets[a].pts, bytes, 1, a, false);
  }
  *total = n;
  return rs.check(fn);
}

// The parameters of cs_rotation_averaging, its host arrays (the outputs R_out, residuals_out, inlier_out, cost_out and
// trace_out share no byte with each other or with the inputs edges, Rrel and weights), then every edge.
int rotavg_args(const char *fn, int numImages, const int *edges, int numEdges, const double *Rrel,
                const double *weights, int refImage, int maxIterations, int maxLinearIterations, double linearTol,
                double sigmaDeg, double maxAngleDeg, const double *R_out, const double *residuals,
                const unsigned char *inlier, const double *cost_out, const double *trace_out)
{
  if (numImages < 1 || numImages > (1 << 24)) return arg_error(fn, "numImages must be in [1, 2^24]");
  if (numEdges < 0 || numEdges > (1 << 26)) return arg_error(fn, "numEdges must be in [0, 2^26]");
  if (refImage < 0 || refImage >= numImages) return arg_error(fn, "refImage must be in [0, numImages)");
  if (maxIterations < 0 || maxIterations > 1000) return arg_error(fn, "maxIterations must be in [0, 1000]");
  if (maxLinearIterations < 1 || maxLinearIterations > 10000)
    return arg_error(fn, "maxLinearIterations must be in [1, 10000]");
  if (!(linearTol > 0.0) || !(linearTol < 1.0)) return arg_error(fn, "linearTol must be in (0, 1)");
  if (!(sigmaDeg >= 0.0) || !(sigmaDeg <= 180.0)) return arg_error(fn, "sigmaDeg must be in [0, 180]");
  if (!(maxAngleDeg > 0.0) || !(maxAngleDeg <= 180.0)) return arg_error(fn, "maxAngleDeg must be in (0, 180]");
  if (numEdges > 0 && (!edges || !Rrel || !weights)) return arg_error(fn, "numEdges > 0 needs edges, Rrel and weights");
  if (!R_out || !cost_out) return arg_error(fn, "R_out and cost_out must not be NULL");
  static const char *const names[8] = {"R_out", "residuals_out", "inlier_out", "cost_out", "trace_out", "edges",
                                        "Rrel", "weights"};
  ArgRanges rs(names, 8);
  const size_t E = (size_t)numEdges;
  rs.add(R_out, (size_t)numImages * 9 * sizeof(double), 0, 0, true);
  if (residuals) rs.add(residuals, E * sizeof(double), 1, 0, true);
  if (inlier) rs.add(inlier, E, 2, 0, true);
  rs.add(cost_out, 2 * sizeof(double), 3, 0, true);
  if (trace_out) rs.add(trace_out, (size_t)maxIterations * 3 * sizeof(double), 4, 0, true);
  if (numEdges > 0) {
    rs.add(edges, E * 2 * sizeof(int), 5, 0, false);
    rs.add(Rrel, E * 9 * sizeof(double), 6, 0, false);
    rs.add(weights, E * sizeof(double), 7, 0, false);
  }
  int r = rs.check(fn);
  if (r < 0) return r;
  for (int e = 0; e < numEdges; e++) {
    const int i = edges[2 * e], j = edges[2 * e + 1];
    if (i < 0 || i >= numImages || j < 0 || j >= numImages)
      return arg_error(fn, "edges[%d] = {%d, %d}: an image index outside [0, numImages)", e, i, j);
    if (i == j) return arg_error(fn, "edges[%d] joins image %d to itself", e, i);
    const double *R = Rrel + 9 * (size_t)e;
    bool ok = true;
    for (int k = 0; k < 9; k++) ok = ok && std::isfinite(R[k]);
    for (int a = 0; a < 3 && ok; a++)
      for (int b = 0; b < 3; b++) {
        const double d = R[a] * R[b] + R[3 + a] * R[3 + b] + R[6 + a] * R[6 + b];
        ok = ok && std::fabs(d - (a == b ? 1.0 : 0.0)) <= 1e-6;
      }
    const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) +
                       R[2] * (R[3] * R[7] - R[4] * R[6]);
    if (!ok || !(std::fabs(det - 1.0) <= 1e-6))
      return arg_error(fn, "Rrel[%d] must be a finite rotation (R^T R = I and det R = 1, within 1e-6)", e);
    if (!std::isfinite(weights[e]) || !(weights[e] > 0.0)) return arg_error(fn, "weights[%d] must be finite and > 0", e);
  }
  return 0;
}

// The images of cs_global_positioning (sets, Ks; Rs[a] a rotation, or all nine entries NaN: not positioned), the
// parameters, then two sweeps: the device ranges (d_points written; d_offsets, d_members, d_use and the records read)
// and the host ranges (t_out, cost_out, trace_out written; Ks and Rs read).
int globalpos_args(const char *fn, const cs_match_set *sets, int numImages, const double *Ks, const double *Rs,
                   const int *offsets, int numTracks, const int *members, int numMembers, const unsigned char *use,
                   int refImage, int loss, double lossScale, int maxIterations, int maxLinearIterations,
                   double linearTol, const double *t_out, const double *points, const double *cost_out,
                   const double *trace_out)
{
  if (numImages < 1 || numImages > (1 << 24)) return arg_error(fn, "numImages must be in [1, 2^24]");
  if (numTracks < 0) return arg_error(fn, "numTracks must be >= 0");
  if (numMembers < 0) return arg_error(fn, "numMembers must be >= 0");
  if (!sets || !Ks || !Rs) return arg_error(fn, "sets, Ks and Rs must not be NULL");
  if (refImage < 0 || refImage >= numImages) return arg_error(fn, "refImage must be in [0, numImages)");
  if (loss < 0 || loss > 2) return arg_error(fn, "loss must be 0 (trivial), 1 (soft-L1) or 2 (Cauchy)");
  if (!std::isfinite(lossScale) || !(lossScale > 0.0)) return arg_error(fn, "lossScale must be finite and > 0");
  if (maxIterations < 0 || maxIterations > 1000) return arg_error(fn, "maxIterations must be in [0, 1000]");
  if (maxLinearIterations < 1 || maxLinearIterations > 10000)
    return arg_error(fn, "maxLinearIterations must be in [1, 10000]");
  if (!(linearTol > 0.0) || !(linearTol < 1.0)) return arg_error(fn, "linearTol must be in (0, 1)");
  if (!t_out || !cost_out) return arg_error(fn, "t_out and cost_out must not be NULL");
  if (numTracks > 0 && (!offsets || !points)) return arg_error(fn, "numTracks > 0 needs d_offsets and d_points");
  if (numMembers > 0 && !members) return arg_error(fn, "numMembers > 0 needs d_members");
  if (misaligned(offsets, 4)) return arg_error(fn, "d_offsets must be 4-byte aligned");
  if (misaligned(members, 8) || misaligned(points, 8))
    return arg_error(fn, "d_members and d_points must be 8-byte aligned");
  int r = check_set_table(fn, sets, numImages);
  if (r < 0) return r;
  for (int a = 0; a < numImages; a++) {
    char name[32];
    snprintf(name, sizeof name, "Ks[%d]", a);
    if ((r = check_intrinsics(fn, Ks + 9 * (size_t)a, name)) < 0) return r;
    const double *R = Rs + 9 * (size_t)a;
    bool nan = true, ok = true;
    for (int k = 0; k < 9; k++) { nan = nan && std::isnan(R[k]); ok = ok && std::isfinite(R[k]); }
    if (nan) continue;
    for (int i = 0; i < 3 && ok; i++)
      for (int j = 0; j < 3; j++) {
        const double d = R[3 * i] * R[3 * j] + R[3 * i + 1] * R[3 * j + 1] + R[3 * i + 2] * R[3 * j + 2];
        ok = ok && std::fabs(d - (i == j ? 1.0 : 0.0)) <= 1e-6;
      }
    const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) +
                       R[2] * (R[3] * R[7] - R[4] * R[6]);
    if (!ok || !(det > 0.0))
      return arg_error(fn, "Rs[%d] must be a rotation (R R^T = I within 1e-6, det R > 0) or all NaN", a);
  }
  static const char *const dnames[5] = {"d_points", "d_offsets", "d_members", "d_use", "sets[%d].pts"};
  ArgRanges rs(dnames, (size_t)numImages + 4);
  if (numTracks > 0) {
    rs.add(points, (size_t)numTracks * 3 * sizeof(double), 0, 0, true);
    rs.add(offsets, ((size_t)numTracks + 1) * sizeof(int), 1, 0, false);
  }
  rs.add(members, (size_t)numMembers * sizeof(int2), 2, 0, false);
  if (use) rs.add(use, (size_t)numMembers, 3, 0, false);
  for (int a = 0; a < numImages; a++) rs.add(sets[a].pts, record_bytes(sets[a].n), 4, a, false);
  if ((r = rs.check(fn)) < 0) return r;
  static const char *const hnames[5] = {"t_out", "cost_out", "trace_out", "Ks", "Rs"};
  ArgRanges hs(hnames, 5);
  hs.add(t_out, (size_t)numImages * 3 * sizeof(double), 0, 0, true);
  hs.add(cost_out, 2 * sizeof(double), 1, 0, true);
  if (trace_out) hs.add(trace_out, (size_t)maxIterations * 4 * sizeof(double), 2, 0, true);
  hs.add(Ks, (size_t)numImages * 9 * sizeof(double), 3, 0, false);
  hs.add(Rs, (size_t)numImages * 9 * sizeof(double), 4, 0, false);
  return hs.check(fn);
}

// The set table of the vocabulary calls and the feature total *M (at most INT_MAX).
static int vocab_sets(const char *fn, const cs_match_set *sets, int numSets, int numWords, int *M)
{
  if (numSets < 0 || numSets > 65536) return arg_error(fn, "numSets must be in [0, 65536]");
  if (numSets > 0 && !sets) return arg_error(fn, "numSets > 0 needs a sets array");
  if (numWords < 1 || numWords > (1 << 18)) return arg_error(fn, "numWords must be in [1, 2^18]");
  int r;
  if ((r = check_set_table(fn, sets, numSets)) < 0) return r;
  long long n = 0;
  for (int s = 0; s < numSets; s++)
    if ((n += sets[s].n) > INT_MAX) return arg_error(fn, "sets[%d]: the set sizes pass INT_MAX", s);
  *M = (int)n;
  return 0;
}

int vocab_assign_args(const char *fn, const cs_match_set *sets, int numSets, const void *vocab, int numWords,
                      const int *wordOf, int *M)
{
  int r;
  if ((r = vocab_sets(fn, sets, numSets, numWords, M)) < 0) return r;
  if (!vocab) return arg_error(fn, "d_vocab must not be NULL");
  if (misaligned(vocab, 16)) return arg_error(fn, "d_vocab must be 16-byte aligned");
  if (*M > 0 && !wordOf) return arg_error(fn, "sets with features need d_wordOf");
  if (misaligned(wordOf, 4)) return arg_error(fn, "d_wordOf must be 4-byte aligned");
  // the output (written), the vocabulary and the records (read)
  static const char *const names[3] = {"d_wordOf", "d_vocab", "sets[%d].pts"};
  ArgRanges rs(names, (size_t)numSets + 2);
  rs.add(wordOf, (size_t)*M * sizeof(int), 0, 0, true);
  rs.add(vocab, record_bytes(numWords), 1, 0, false);
  for (int s = 0; s < numSets; s++) rs.add(sets[s].pts, record_bytes(sets[s].n), 2, s, false);
  return rs.check(fn);
}

int vocab_train_args(const char *fn, const cs_match_set *sets, int numSets, int numWords, int maxIterations,
                     const void *vocab, int *M)
{
  int r;
  if ((r = vocab_sets(fn, sets, numSets, numWords, M)) < 0) return r;
  if (numWords > *M) return arg_error(fn, "numWords must not exceed the feature count (%d)", *M);
  if (maxIterations < 0 || maxIterations > 1000) return arg_error(fn, "maxIterations must be in [0, 1000]");
  if (!vocab) return arg_error(fn, "d_vocab must not be NULL");
  if (misaligned(vocab, 16)) return arg_error(fn, "d_vocab must be 16-byte aligned");
  static const char *const names[2] = {"d_vocab", "sets[%d].pts"};
  ArgRanges rs(names, (size_t)numSets + 1);
  rs.add(vocab, record_bytes(numWords), 0, 0, true);
  for (int s = 0; s < numSets; s++) rs.add(sets[s].pts, record_bytes(sets[s].n), 1, s, false);
  return rs.check(fn);
}

int retrieve_args(const char *fn, const int *imageSizes, int numImages, const int *wordOf, int numWords, int topK,
                  const int *neighbours, const double *scores, const double *idf, const int *pairs, int maxPairs,
                  int *N)
{
  if (numImages < 0 || numImages > 65536) return arg_error(fn, "numImages must be in [0, 65536]");
  if (numImages > 0 && !imageSizes) return arg_error(fn, "numImages > 0 needs an imageSizes array");
  long long n = 0;
  for (int a = 0; a < numImages; a++) {
    if (imageSizes[a] < 0) return arg_error(fn, "imageSizes[%d] must be >= 0", a);
    if ((n += imageSizes[a]) > INT_MAX) return arg_error(fn, "imageSizes[%d]: the sizes pass INT_MAX", a);
  }
  if (numWords < 1 || numWords > (1 << 18)) return arg_error(fn, "numWords must be in [1, 2^18]");
  if (topK < 1 || topK > 1024) return arg_error(fn, "topK must be in [1, 1024]");
  if (maxPairs < 0) return arg_error(fn, "maxPairs must be >= 0");
  if (n > 0 && !wordOf) return arg_error(fn, "images with features need d_wordOf");
  if (numImages > 0 && (!neighbours || !scores)) return arg_error(fn, "numImages > 0 needs d_neighbours and d_scores");
  if (maxPairs > 0 && !pairs) return arg_error(fn, "maxPairs > 0 needs d_pairs");
  if (misaligned(wordOf, 4) || misaligned(neighbours, 4))
    return arg_error(fn, "d_wordOf and d_neighbours must be 4-byte aligned");
  if (misaligned(scores, 8) || misaligned(idf, 8) || misaligned(pairs, 8))
    return arg_error(fn, "d_scores, d_idf and d_pairs must be 8-byte aligned");
  // the outputs (written) and the words (read)
  static const char *const names[5] = {"d_wordOf", "d_neighbours", "d_scores", "d_idf", "d_pairs"};
  ArgRanges rs(names, 5);
  const size_t lists = (size_t)numImages * topK;
  rs.add(wordOf, (size_t)n * sizeof(int), 0, 0, false);
  rs.add(neighbours, lists * sizeof(int), 1, 0, true);
  rs.add(scores, lists * sizeof(double), 2, 0, true);
  if (idf) rs.add(idf, (size_t)numWords * sizeof(double), 3, 0, true);
  rs.add(pairs, (size_t)maxPairs * sizeof(int2), 4, 0, true);
  *N = (int)n;
  return rs.check(fn);
}

// The counts and tables, every job (named jobs[p]) and its K, the parameters, then every per-feature output against
// the other outputs, every record range, every pointOf and the points.  Jobs with n <= 0 have no ranges.
int pose_args(const char *fn, const double *points, int numPoints, const cs_pose_job *jobs, int numJobs,
              const double *Ks, int numLoops, double maxError)
{
  if (numJobs < 0 || numJobs > 65536) return arg_error(fn, "numJobs must be in [0, 65536]");
  if (numJobs > 0 && (!jobs || !Ks)) return arg_error(fn, "numJobs > 0 needs jobs and Ks");
  if (numPoints < 0) return arg_error(fn, "numPoints must be >= 0");
  if (numPoints > 0 && !points) return arg_error(fn, "numPoints > 0 needs d_points");
  if (misaligned(points, 8)) return arg_error(fn, "d_points must be 8-byte aligned");
  for (int p = 0; p < numJobs; p++) {
    const cs_pose_job &j = jobs[p];
    if (j.n < 0) return arg_error(fn, "jobs[%d]: n must be >= 0", p);
    if (j.n > 0 && (!j.pts || !j.pointOf)) return arg_error(fn, "jobs[%d]: n > 0 needs pts and pointOf", p);
    if (misaligned(j.pointOf, 4) || misaligned(j.errors, 4))
      return arg_error(fn, "jobs[%d]: pointOf and errors must be 4-byte aligned", p);
  }
  for (int p = 0; p < numJobs; p++) {
    char name[96];
    snprintf(name, sizeof name, "%s: jobs[%d]", fn, p);
    const int r = check_intrinsics(name, Ks + 9 * (size_t)p, "Ks[p]");
    if (r < 0) return r;
  }
  if (numLoops < 1 || numLoops > 65536) return arg_error(fn, "numLoops must be in [1, 65536]");
  if (!std::isfinite(maxError) || !(maxError > 0.0)) return arg_error(fn, "maxError must be finite and > 0");
  // the per-feature outputs (written), the records, pointOf and the points (read)
  static const char *const names[5] = {"jobs[%d].errors", "jobs[%d].inlier", "jobs[%d].pts", "jobs[%d].pointOf",
                                       "d_points"};
  ArgRanges rs(names, 4 * (size_t)numJobs + 1);
  for (int p = 0; p < numJobs; p++) {
    const cs_pose_job &j = jobs[p];
    if (j.n <= 0) continue;
    if (j.errors) rs.add(j.errors, (size_t)j.n * sizeof(float), 0, p, true);
    if (j.inlier) rs.add(j.inlier, (size_t)j.n, 1, p, true);
    rs.add(j.pts, record_bytes(j.n), 2, p, false);
    rs.add(j.pointOf, (size_t)j.n * sizeof(int), 3, p, false);
  }
  rs.add(points, (size_t)numPoints * 3 * sizeof(double), 4, 0, false);
  return rs.check(fn);
}

// ---- dense reconstruction -------------------------------------------------------------------------------------------

// The bytes an image's rows span.
static size_t image_bytes(const cs_image &I) { return ((size_t)(I.height - 1) * I.pitch + I.width) * sizeof(float); }

// The images and cameras of the dense calls (Rs and ts only with poses): numImages in [lo, 65536].
static int stereo_images(const char *fn, const cs_image *images, int numImages, int lo, const double *Ks,
                         const double *Rs, const double *ts, bool poses)
{
  if (numImages < lo || numImages > 65536) return arg_error(fn, "numImages must be in [%d, 65536]", lo);
  if (numImages > 0 && (!images || !Ks || (poses && (!Rs || !ts))))
    return arg_error(fn, poses ? "images, Ks, Rs and ts must not be NULL" : "images and Ks must not be NULL");
  for (int a = 0; a < numImages; a++) {
    const cs_image &I = images[a];
    if (!I.d_img || misaligned(I.d_img, 4)) return arg_error(fn, "images[%d].d_img must be a 4-byte aligned pointer", a);
    if (I.width < 2 || I.width > 4096 || I.height < 2 || I.height > 4096)
      return arg_error(fn, "images[%d]: width and height must be in [2, 4096]", a);
    if (I.pitch < I.width) return arg_error(fn, "images[%d]: pitch must be >= width", a);
    char name[32];
    snprintf(name, sizeof name, "Ks[%d]", a);
    int r;
    if ((r = check_intrinsics(fn, Ks + 9 * (size_t)a, name)) < 0) return r;
    if (!poses) continue;
    const double *R = Rs + 9 * (size_t)a, *t = ts + 3 * (size_t)a;
    bool ok = true;
    for (int k = 0; k < 9; k++) ok = ok && std::isfinite(R[k]);
    for (int i = 0; i < 3 && ok; i++)
      for (int j = 0; j < 3; j++) {
        const double d = R[3 * i] * R[3 * j] + R[3 * i + 1] * R[3 * j + 1] + R[3 * i + 2] * R[3 * j + 2];
        ok = ok && std::fabs(d - (i == j ? 1.0 : 0.0)) <= 1e-6;
      }
    const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) +
                       R[2] * (R[3] * R[7] - R[4] * R[6]);
    if (!ok || !(det > 0.0)) return arg_error(fn, "Rs[%d] must be a rotation (R R^T = I within 1e-6, det R > 0)", a);
    if (!std::isfinite(t[0]) || !std::isfinite(t[1]) || !std::isfinite(t[2]))
      return arg_error(fn, "ts[%d] must be finite", a);
  }
  return 0;
}

int undistort_images_args(const char *fn, const cs_image *images, int numImages, const double *Ks,
                          const double *dists, float *const *d_out)
{
  int r;
  if ((r = stereo_images(fn, images, numImages, 0, Ks, nullptr, nullptr, false)) < 0) return r;
  if (numImages > 0 && !d_out) return arg_error(fn, "numImages > 0 needs d_out");
  for (int a = 0; a < numImages; a++) {
    if (dists && (!std::isfinite(dists[2 * (size_t)a]) || !std::isfinite(dists[2 * (size_t)a + 1])))
      return arg_error(fn, "dists[%d] must be finite", a);
    if (!d_out[a] || misaligned(d_out[a], 4)) return arg_error(fn, "d_out[%d] must be a 4-byte aligned pointer", a);
  }
  // the outputs (written) and the images (read)
  static const char *const names[2] = {"d_out[%d]", "images[%d].d_img"};
  ArgRanges rs(names, 2 * (size_t)numImages);
  for (int a = 0; a < numImages; a++) {
    rs.add(d_out[a], (size_t)images[a].width * images[a].height * sizeof(float), 0, a, true);
    rs.add(images[a].d_img, image_bytes(images[a]), 1, a, false);
  }
  return rs.check(fn);
}

// The jobs of the dense calls (topK checked when > 0); *pixels receives the pixels of all jobs.
static int stereo_jobs(const char *fn, int numImages, const cs_image *images, const cs_stereo_job *jobs, int numJobs,
                       int topK, long long *pixels)
{
  if (numJobs < 0 || numJobs > 65536) return arg_error(fn, "numJobs must be in [0, 65536]");
  if (numJobs > 0 && !jobs) return arg_error(fn, "numJobs > 0 needs jobs");
  std::vector<int> refOf(numImages, -1);
  long long n = 0;
  for (int p = 0; p < numJobs; p++) {
    const cs_stereo_job &J = jobs[p];
    if (J.ref < 0 || J.ref >= numImages) return arg_error(fn, "jobs[%d]: ref must be in [0, numImages)", p);
    if (refOf[J.ref] >= 0) return arg_error(fn, "jobs[%d]: image %d is already the ref of jobs[%d]", p, J.ref, refOf[J.ref]);
    refOf[J.ref] = p;
    if (J.numSources < 1 || J.numSources > 32) return arg_error(fn, "jobs[%d]: numSources must be in [1, 32]", p);
    if (!J.sources) return arg_error(fn, "jobs[%d]: sources must not be NULL", p);
    for (int s = 0; s < J.numSources; s++) {
      const int b = J.sources[s];
      if (b < 0 || b >= numImages || b == J.ref)
        return arg_error(fn, "jobs[%d]: sources[%d] must be in [0, numImages) and not ref", p, s);
      for (int u = 0; u < s; u++)
        if (J.sources[u] == b) return arg_error(fn, "jobs[%d]: sources[%d] repeats sources[%d]", p, s, u);
    }
    if (topK > 0 && topK > J.numSources) return arg_error(fn, "jobs[%d]: topK must be in [1, numSources]", p);
    if (!std::isfinite(J.depthMin) || !std::isfinite(J.depthMax) || !(J.depthMin > 0.0f) ||
        !(J.depthMin < J.depthMax))
      return arg_error(fn, "jobs[%d]: depthMin and depthMax must be finite with 0 < depthMin < depthMax", p);
    if (!J.d_depth || !J.d_normal || !J.d_cost || misaligned(J.d_depth, 4) || misaligned(J.d_normal, 4) ||
        misaligned(J.d_cost, 4))
      return arg_error(fn, "jobs[%d]: d_depth, d_normal and d_cost must be 4-byte aligned pointers", p);
    n += (long long)images[J.ref].width * images[J.ref].height;
  }
  *pixels = n;
  return 0;
}

// The maps (kinds 0..2, written when mapsWritten) and the images (kind 3) of a dense call.
static void stereo_ranges(ArgRanges &rs, const cs_image *images, int numImages, const cs_stereo_job *jobs,
                          int numJobs, bool mapsWritten, int kind0)
{
  for (int p = 0; p < numJobs; p++) {
    const cs_image &I = images[jobs[p].ref];
    const size_t px = (size_t)I.width * I.height * sizeof(float);
    rs.add(jobs[p].d_depth, px, kind0, p, mapsWritten);
    rs.add(jobs[p].d_normal, 3 * px, kind0 + 1, p, mapsWritten);
    rs.add(jobs[p].d_cost, px, kind0 + 2, p, mapsWritten);
  }
  for (int a = 0; a < numImages; a++) rs.add(images[a].d_img, image_bytes(images[a]), kind0 + 3, a, false);
}

// The checks of the PatchMatch calls before their range sweeps; numIterations in [0, maxIterations].
static int pm_args(const char *fn, const cs_image *images, int numImages, const double *Ks, const double *Rs,
                   const double *ts, const cs_stereo_job *jobs, int numJobs, int windowRadius, int windowStep,
                   int numIterations, int maxIterations, int topK)
{
  int r;
  if ((r = stereo_images(fn, images, numImages, 1, Ks, Rs, ts, true)) < 0) return r;
  if (windowRadius < 1 || windowRadius > 7) return arg_error(fn, "windowRadius must be in [1, 7]");
  if (windowStep < 1 || windowStep > windowRadius || windowRadius % windowStep != 0)
    return arg_error(fn, "windowStep must be in [1, windowRadius] and divide windowRadius");
  if (numIterations < 0 || numIterations > maxIterations)
    return arg_error(fn, "numIterations must be in [0, %d]", maxIterations);
  if (topK < 1) return arg_error(fn, "topK must be in [1, numSources]");
  long long pixels = 0;
  return stereo_jobs(fn, numImages, images, jobs, numJobs, topK, &pixels);
}

int patch_match_args(const char *fn, const cs_image *images, int numImages, const double *Ks, const double *Rs,
                     const double *ts, const cs_stereo_job *jobs, int numJobs, int windowRadius, int windowStep,
                     int numIterations, int topK)
{
  int r;
  if ((r = pm_args(fn, images, numImages, Ks, Rs, ts, jobs, numJobs, windowRadius, windowStep, numIterations, 32,
                   topK)) < 0)
    return r;
  static const char *const names[4] = {"jobs[%d].d_depth", "jobs[%d].d_normal", "jobs[%d].d_cost",
                                       "images[%d].d_img"};
  ArgRanges rs(names, 3 * (size_t)numJobs + numImages);
  stereo_ranges(rs, images, numImages, jobs, numJobs, true, 0);
  return rs.check(fn);
}

// The draws of the geometric pass use counter iterations 32 + k, within the counter's 6 bits: at most 31 iterations.
int patch_match_geometric_args(const char *fn, const cs_image *images, int numImages, const double *Ks,
                               const double *Rs, const double *ts, const cs_depth_prior *priors,
                               const cs_stereo_job *jobs, int numJobs, int windowRadius, int windowStep,
                               int numIterations, int topK, double geomWeight, double geomMaxError)
{
  int r;
  if ((r = pm_args(fn, images, numImages, Ks, Rs, ts, jobs, numJobs, windowRadius, windowStep, numIterations, 31,
                   topK)) < 0)
    return r;
  if (numJobs > 0 && !priors) return arg_error(fn, "numJobs > 0 needs priors");
  for (int p = 0; p < numJobs; p++) {
    const cs_depth_prior &Pr = priors[jobs[p].ref];
    if (!Pr.d_depth || !Pr.d_normal)
      return arg_error(fn, "jobs[%d]: priors[%d] (its ref) needs d_depth and d_normal", p, jobs[p].ref);
  }
  for (int a = 0; priors && a < numImages; a++)
    if (misaligned(priors[a].d_depth, 4) || misaligned(priors[a].d_normal, 4))
      return arg_error(fn, "priors[%d]: d_depth and d_normal must be 4-byte aligned", a);
  if (!std::isfinite(geomWeight) || !(geomWeight >= 0.0)) return arg_error(fn, "geomWeight must be finite and >= 0");
  if (!std::isfinite(geomMaxError) || !(geomMaxError > 0.0))
    return arg_error(fn, "geomMaxError must be finite and > 0");
  // the maps (written), the images and the priors (read, so they may share bytes with each other)
  static const char *const names[6] = {"jobs[%d].d_depth", "jobs[%d].d_normal", "jobs[%d].d_cost",
                                       "images[%d].d_img", "priors[%d].d_depth", "priors[%d].d_normal"};
  ArgRanges rs(names, 3 * (size_t)numJobs + 3 * (size_t)numImages);
  stereo_ranges(rs, images, numImages, jobs, numJobs, true, 0);
  for (int a = 0; priors && a < numImages; a++) {
    const size_t px = (size_t)images[a].width * images[a].height * sizeof(float);
    if (priors[a].d_depth) rs.add(priors[a].d_depth, px, 4, a, false);
    if (priors[a].d_normal) rs.add(priors[a].d_normal, 3 * px, 5, a, false);
  }
  return rs.check(fn);
}

int fuse_args(const char *fn, const cs_image *images, int numImages, const double *Ks, const double *Rs,
              const double *ts, const cs_stereo_job *jobs, int numJobs, float maxCost, int minConsistent,
              double maxReprojError, double maxDepthError, double maxNormalErrorDeg, const float *xyz,
              const float *normal, const float *intensity, const int *source, int maxPoints)
{
  int r;
  if ((r = stereo_images(fn, images, numImages, 1, Ks, Rs, ts, true)) < 0) return r;
  long long pixels = 0;
  if ((r = stereo_jobs(fn, numImages, images, jobs, numJobs, 0, &pixels)) < 0) return r;
  if (pixels > INT_MAX) return arg_error(fn, "the pixels of all jobs must be at most 2^31 - 1");
  if (!(maxCost >= 0.0f && maxCost <= 2.0f)) return arg_error(fn, "maxCost must be in [0, 2]");
  if (minConsistent < 1 || minConsistent > 32) return arg_error(fn, "minConsistent must be in [1, 32]");
  if (!std::isfinite(maxReprojError) || !(maxReprojError > 0.0))
    return arg_error(fn, "maxReprojError must be finite and > 0");
  if (!std::isfinite(maxDepthError) || !(maxDepthError > 0.0))
    return arg_error(fn, "maxDepthError must be finite and > 0");
  if (!(maxNormalErrorDeg > 0.0 && maxNormalErrorDeg <= 180.0))
    return arg_error(fn, "maxNormalErrorDeg must be in (0, 180]");
  if (maxPoints < 0) return arg_error(fn, "maxPoints must be >= 0");
  if (maxPoints > 0 && (!xyz || !normal || !intensity || !source || misaligned(xyz, 4) || misaligned(normal, 4) ||
                        misaligned(intensity, 4) || misaligned(source, 8)))
    return arg_error(fn, "maxPoints > 0 needs d_xyz, d_normal, d_intensity (4-byte aligned) and d_source (8-byte)");
  static const char *const names[8] = {"d_xyz", "d_normal", "d_intensity", "d_source", "jobs[%d].d_depth",
                                       "jobs[%d].d_normal", "jobs[%d].d_cost", "images[%d].d_img"};
  ArgRanges rs(names, 4 + 3 * (size_t)numJobs + numImages);
  if (maxPoints > 0) {
    const size_t m = (size_t)maxPoints;
    rs.add(xyz, 12 * m, 0, 0, true);
    rs.add(normal, 12 * m, 1, 0, true);
    rs.add(intensity, 4 * m, 2, 0, true);
    rs.add(source, 8 * m, 3, 0, true);
  }
  stereo_ranges(rs, images, numImages, jobs, numJobs, false, 4);
  return rs.check(fn);
}

int mesh_args(const char *fn, const float *xyz, const float *normal, const float *intensity, int numPoints, int depth,
              double scale, int maxIterations, double tol, double trim, const float *vertices,
              const float *vertexIntensity, int maxVertices, const int *triangles, int maxTriangles, const float *chi)
{
  if (numPoints < 0 || numPoints > (1 << 30)) return arg_error(fn, "numPoints must be in [0, 2^30]");
  if (depth < 4 || depth > 9) return arg_error(fn, "depth must be in [4, 9]");
  if (!std::isfinite(scale) || scale < 1.0 || scale > 4.0) return arg_error(fn, "scale must be finite and in [1, 4]");
  if (maxIterations < 1 || maxIterations > 1000) return arg_error(fn, "maxIterations must be in [1, 1000]");
  if (!(tol > 0.0 && tol < 1.0)) return arg_error(fn, "tol must be in (0, 1)");
  if (!std::isfinite(trim) || trim < 0.0) return arg_error(fn, "trim must be finite and >= 0");
  if (maxVertices < 0) return arg_error(fn, "maxVertices must be >= 0");
  if (maxTriangles < 0) return arg_error(fn, "maxTriangles must be >= 0");
  if (numPoints > 0 && (!xyz || misaligned(xyz, 4)))
    return arg_error(fn, "numPoints > 0 needs d_xyz (4-byte aligned)");
  if (numPoints > 0 && (!normal || misaligned(normal, 4)))
    return arg_error(fn, "numPoints > 0 needs d_normal (4-byte aligned)");
  if (maxVertices > 0 && (!vertices || misaligned(vertices, 4)))
    return arg_error(fn, "maxVertices > 0 needs d_vertices (4-byte aligned)");
  if (maxTriangles > 0 && (!triangles || misaligned(triangles, 4)))
    return arg_error(fn, "maxTriangles > 0 needs d_triangles (4-byte aligned)");
  if (misaligned(intensity, 4)) return arg_error(fn, "d_intensity must be 4-byte aligned");
  if (misaligned(vertexIntensity, 4)) return arg_error(fn, "d_vertexIntensity must be 4-byte aligned");
  if (misaligned(chi, 4)) return arg_error(fn, "d_chi must be 4-byte aligned");
  if (!intensity != !vertexIntensity)
    return arg_error(fn, "d_intensity and d_vertexIntensity must be given together or not at all");
  static const char *const names[7] = {"d_vertices", "d_vertexIntensity", "d_triangles", "d_chi",
                                       "d_xyz", "d_normal", "d_intensity"};
  ArgRanges rs(names, 7);
  const size_t n1 = ((size_t)1 << depth) + 1, P = (size_t)numPoints, V = (size_t)maxVertices;
  rs.add(vertices, 12 * V, 0, 0, true);
  if (vertexIntensity) rs.add(vertexIntensity, 4 * V, 1, 0, true);
  rs.add(triangles, 12 * (size_t)maxTriangles, 2, 0, true);
  if (chi) rs.add(chi, 4 * n1 * n1 * n1, 3, 0, true);
  rs.add(xyz, 12 * P, 4, 0, false);
  rs.add(normal, 12 * P, 5, 0, false);
  if (intensity) rs.add(intensity, 4 * P, 6, 0, false);
  return rs.check(fn);
}

int mesh_screened_args(const char *fn, const float *xyz, const float *normal, const float *intensity, int numPoints,
                       int depth, double scale, double pointWeight, int maxIterations, double tol, double trim,
                       const float *vertices, const float *vertexIntensity, int maxVertices, const int *triangles,
                       int maxTriangles, const float *chi)
{
  if (!std::isfinite(pointWeight) || pointWeight <= 0.0 || pointWeight > 1000.0)
    return arg_error(fn, "pointWeight must be finite and in (0, 1000]");
  return mesh_args(fn, xyz, normal, intensity, numPoints, depth, scale, maxIterations, tol, trim, vertices,
                   vertexIntensity, maxVertices, triangles, maxTriangles, chi);
}

int simplify_args(const char *fn, const float *vertices, const float *vertexIntensity, int numVertices,
                  const int *triangles, int numTriangles, int targetTriangles, double maxError, double boundaryWeight,
                  const float *outVertices, const float *outIntensity, int maxOutVertices, const int *outTriangles,
                  int maxOutTriangles)
{
  if (numVertices < 0 || numVertices > (1 << 30)) return arg_error(fn, "numVertices must be in [0, 2^30]");
  if (numTriangles < 0 || numTriangles > (1 << 29)) return arg_error(fn, "numTriangles must be in [0, 2^29]");
  if (targetTriangles < 0) return arg_error(fn, "targetTriangles must be >= 0");
  if (!(maxError >= 0.0)) return arg_error(fn, "maxError must be >= 0 (inf allowed)");
  if (!std::isfinite(boundaryWeight) || boundaryWeight < 0.0)
    return arg_error(fn, "boundaryWeight must be finite and >= 0");
  if (maxOutVertices < 0) return arg_error(fn, "maxOutVertices must be >= 0");
  if (maxOutTriangles < 0) return arg_error(fn, "maxOutTriangles must be >= 0");
  if (numVertices > 0 && (!vertices || misaligned(vertices, 4)))
    return arg_error(fn, "numVertices > 0 needs d_vertices (4-byte aligned)");
  if (numTriangles > 0 && (!triangles || misaligned(triangles, 4)))
    return arg_error(fn, "numTriangles > 0 needs d_triangles (4-byte aligned)");
  if (maxOutVertices > 0 && (!outVertices || misaligned(outVertices, 4)))
    return arg_error(fn, "maxOutVertices > 0 needs d_outVertices (4-byte aligned)");
  if (maxOutTriangles > 0 && (!outTriangles || misaligned(outTriangles, 4)))
    return arg_error(fn, "maxOutTriangles > 0 needs d_outTriangles (4-byte aligned)");
  if (misaligned(vertexIntensity, 4)) return arg_error(fn, "d_vertexIntensity must be 4-byte aligned");
  if (misaligned(outIntensity, 4)) return arg_error(fn, "d_outIntensity must be 4-byte aligned");
  if (!vertexIntensity != !outIntensity)
    return arg_error(fn, "d_vertexIntensity and d_outIntensity must be given together or not at all");
  static const char *const names[6] = {"d_outVertices", "d_outIntensity", "d_outTriangles",
                                       "d_vertices", "d_vertexIntensity", "d_triangles"};
  ArgRanges rs(names, 6);
  const size_t V = (size_t)numVertices, W = (size_t)maxOutVertices;
  rs.add(outVertices, 12 * W, 0, 0, true);
  if (outIntensity) rs.add(outIntensity, 4 * W, 1, 0, true);
  rs.add(outTriangles, 12 * (size_t)maxOutTriangles, 2, 0, true);
  rs.add(vertices, 12 * V, 3, 0, false);
  if (vertexIntensity) rs.add(vertexIntensity, 4 * V, 4, 0, false);
  rs.add(triangles, 12 * (size_t)numTriangles, 5, 0, false);
  return rs.check(fn);
}

int clean_args(const char *fn, const float *vertices, const float *vertexIntensity, int numVertices,
               const int *triangles, int numTriangles, int removeDegenerate, double longEdgeFactor,
               int removeNonManifold, int minComponentFaces, double minComponentFraction, int maxHoleEdges,
               int smoothIterations, double lambda, double mu, const float *outVertices, const float *outIntensity,
               int maxOutVertices, const int *outTriangles, int maxOutTriangles)
{
  if (numTriangles < 0 || numTriangles > (1 << 26)) return arg_error(fn, "numTriangles must be in [0, 2^26]");
  if (removeDegenerate != 0 && removeDegenerate != 1) return arg_error(fn, "removeDegenerate must be 0 or 1");
  if (!std::isfinite(longEdgeFactor) || longEdgeFactor < 0.0)
    return arg_error(fn, "longEdgeFactor must be finite and >= 0");
  if (removeNonManifold != 0 && removeNonManifold != 1) return arg_error(fn, "removeNonManifold must be 0 or 1");
  if (minComponentFaces < 0) return arg_error(fn, "minComponentFaces must be >= 0");
  if (!(minComponentFraction >= 0.0 && minComponentFraction <= 1.0))
    return arg_error(fn, "minComponentFraction must be in [0, 1]");
  if (maxHoleEdges != 0 && (maxHoleEdges < 3 || maxHoleEdges > 256))
    return arg_error(fn, "maxHoleEdges must be 0 or in [3, 256]");
  if (smoothIterations < 0 || smoothIterations > 1000) return arg_error(fn, "smoothIterations must be in [0, 1000]");
  if (!(lambda > 0.0 && lambda <= 1.0)) return arg_error(fn, "lambda must be in (0, 1]");
  if (!(mu >= -1.0 && mu < 0.0)) return arg_error(fn, "mu must be in [-1, 0)");
  return simplify_args(fn, vertices, vertexIntensity, numVertices, triangles, numTriangles, 0, 0.0, 0.0, outVertices,
                       outIntensity, maxOutVertices, outTriangles, maxOutTriangles);
}

int texture_args(const char *fn, const cs_image *images, int numImages, const double *Ks, const double *Rs,
                 const double *ts, const float *vertices, int numVertices, const int *triangles, int numTriangles,
                 double lambda, double maxViewAngleDeg, double depthTol, int padding, int atlasWidth, int maxSweeps,
                 const float *atlas, int maxAtlasRows, const float *uv, const int *faceView, const int *faceChart,
                 const int *chartsOut, int maxCharts)
{
  int r;
  if ((r = stereo_images(fn, images, numImages, 1, Ks, Rs, ts, true)) < 0) return r;
  if (numVertices < 0 || numVertices > (1 << 30)) return arg_error(fn, "numVertices must be in [0, 2^30]");
  if (numTriangles < 0 || numTriangles > (1 << 29)) return arg_error(fn, "numTriangles must be in [0, 2^29]");
  if (!std::isfinite(lambda) || lambda < 0.0) return arg_error(fn, "lambda must be finite and >= 0");
  if (!(maxViewAngleDeg > 0.0 && maxViewAngleDeg <= 90.0)) return arg_error(fn, "maxViewAngleDeg must be in (0, 90]");
  if (!(depthTol >= 0.0 && depthTol <= 1.0)) return arg_error(fn, "depthTol must be finite and in [0, 1]");
  if (padding < 0 || padding > 16) return arg_error(fn, "padding must be in [0, 16]");
  int widest = 0;
  for (int a = 0; a < numImages; a++) widest = std::max(widest, images[a].width);
  if (atlasWidth < widest || atlasWidth > 32768)
    return arg_error(fn, "atlasWidth must be in [the largest image width (%d), 32768]", widest);
  if (maxSweeps < 0 || maxSweeps > 1000) return arg_error(fn, "maxSweeps must be in [0, 1000]");
  if (maxAtlasRows < 0) return arg_error(fn, "maxAtlasRows must be >= 0");
  if (maxCharts < 0) return arg_error(fn, "maxCharts must be >= 0");
  if (numVertices > 0 && (!vertices || misaligned(vertices, 4)))
    return arg_error(fn, "numVertices > 0 needs d_vertices (4-byte aligned)");
  if (numTriangles > 0 && (!triangles || misaligned(triangles, 4)))
    return arg_error(fn, "numTriangles > 0 needs d_triangles (4-byte aligned)");
  if (numTriangles > 0 && (!uv || misaligned(uv, 4)))
    return arg_error(fn, "numTriangles > 0 needs d_uv (4-byte aligned)");
  if (numTriangles > 0 && (!faceView || misaligned(faceView, 4)))
    return arg_error(fn, "numTriangles > 0 needs d_faceView (4-byte aligned)");
  if (misaligned(faceChart, 4)) return arg_error(fn, "d_faceChart must be 4-byte aligned");
  if (maxAtlasRows > 0 && (!atlas || misaligned(atlas, 4)))
    return arg_error(fn, "maxAtlasRows > 0 needs d_atlas (4-byte aligned)");
  if (maxCharts > 0 && !chartsOut) return arg_error(fn, "maxCharts > 0 needs charts_out");
  // the outputs (written), the mesh and the images (read)
  static const char *const names[7] = {"d_atlas", "d_uv", "d_faceView", "d_faceChart",
                                       "d_vertices", "d_triangles", "images[%d].d_img"};
  ArgRanges rs(names, 6 + (size_t)numImages);
  const size_t T = (size_t)numTriangles;
  rs.add(atlas, 4 * (size_t)maxAtlasRows * atlasWidth, 0, 0, true);
  rs.add(uv, 24 * T, 1, 0, true);
  rs.add(faceView, 4 * T, 2, 0, true);
  if (faceChart) rs.add(faceChart, 4 * T, 3, 0, true);
  rs.add(vertices, 12 * (size_t)numVertices, 4, 0, false);
  rs.add(triangles, 12 * T, 5, 0, false);
  for (int a = 0; a < numImages; a++) rs.add(images[a].d_img, image_bytes(images[a]), 6, a, false);
  return rs.check(fn);
}

int texture_photo_args(const char *fn, int dataTerm, double outlierK, double outlierMinSigma)
{
  if (dataTerm != 0 && dataTerm != 1) return arg_error(fn, "dataTerm must be 0 (area) or 1 (GMI)");
  if (!(outlierK == 0.0 || (outlierK >= 1.0 && outlierK <= 100.0)))
    return arg_error(fn, "outlierK must be 0 or in [1, 100]");
  if (!(outlierMinSigma > 0.0 && outlierMinSigma <= 1000.0))
    return arg_error(fn, "outlierMinSigma must be finite and in (0, 1000]");
  return 0;
}

int texture_bp_args(const char *fn, int maxBpSweeps)
{
  if (maxBpSweeps < 0 || maxBpSweeps > 1000) return arg_error(fn, "maxBpSweeps must be in [0, 1000]");
  return 0;
}

int refine_args(const char *fn, const cs_image *images, int numImages, const double *Ks, const double *Rs,
                const double *ts, const float *vertices, int numVertices, const int *triangles, int numTriangles,
                const int *pairs, int numPairs, int windowRadius, double smoothness, double step, int maxIterations,
                double depthTol, const float *outVertices)
{
  int r;
  if ((r = stereo_images(fn, images, numImages, 1, Ks, Rs, ts, true)) < 0) return r;
  if (numVertices < 0 || numVertices > (1 << 30)) return arg_error(fn, "numVertices must be in [0, 2^30]");
  if (numTriangles < 0 || numTriangles > (1 << 28)) return arg_error(fn, "numTriangles must be in [0, 2^28]");
  if (numPairs < 0) return arg_error(fn, "numPairs must be >= 0");
  if (numPairs > 0 && !pairs) return arg_error(fn, "numPairs > 0 needs pairs");
  for (int q = 0; q < numPairs; q++) {
    const int a = pairs[2 * q], b = pairs[2 * q + 1];
    if (a < 0 || a >= numImages || b < 0 || b >= numImages)
      return arg_error(fn, "pairs[%d] = {%d, %d} names an image outside [0, %d)", q, a, b, numImages);
    if (a == b) return arg_error(fn, "pairs[%d] has ref == src (%d)", q, a);
  }
  if (windowRadius < 1 || windowRadius > 5) return arg_error(fn, "windowRadius must be in [1, 5]");
  if (!std::isfinite(smoothness) || smoothness < 0.0) return arg_error(fn, "smoothness must be finite and >= 0");
  if (!(step > 0.0 && step <= 1.0)) return arg_error(fn, "step must be in (0, 1]");
  if (maxIterations < 0 || maxIterations > 1000) return arg_error(fn, "maxIterations must be in [0, 1000]");
  if (!(depthTol >= 0.0 && depthTol <= 1.0)) return arg_error(fn, "depthTol must be finite and in [0, 1]");
  if (numVertices > 0 && (!vertices || misaligned(vertices, 4)))
    return arg_error(fn, "numVertices > 0 needs d_vertices (4-byte aligned)");
  if (numVertices > 0 && (!outVertices || misaligned(outVertices, 4)))
    return arg_error(fn, "numVertices > 0 needs d_outVertices (4-byte aligned)");
  if (numTriangles > 0 && (!triangles || misaligned(triangles, 4)))
    return arg_error(fn, "numTriangles > 0 needs d_triangles (4-byte aligned)");
  // the output (written), the mesh and the images (read)
  static const char *const names[4] = {"d_outVertices", "d_vertices", "d_triangles", "images[%d].d_img"};
  ArgRanges rs(names, 3 + (size_t)numImages);
  rs.add(outVertices, 12 * (size_t)numVertices, 0, 0, true);
  rs.add(vertices, 12 * (size_t)numVertices, 1, 0, false);
  rs.add(triangles, 12 * (size_t)numTriangles, 2, 0, false);
  for (int a = 0; a < numImages; a++) rs.add(images[a].d_img, image_bytes(images[a]), 3, a, false);
  return rs.check(fn);
}

int seams_args(const char *fn, const float *vertices, int numVertices, const int *triangles, int numTriangles,
               const int *faceView, const float *uv, const int *charts, int numCharts, const float *atlas,
               int atlasRows, int atlasWidth, int padding, double smoothness, double regularization, bool local,
               int stripWidth, int maxIterations, double tol, const float *outAtlas, const float *cornerOffset)
{
  if (numVertices < 0 || numVertices > (1 << 30)) return arg_error(fn, "numVertices must be in [0, 2^30]");
  if (numTriangles < 0 || numTriangles > (1 << 29)) return arg_error(fn, "numTriangles must be in [0, 2^29]");
  if (atlasRows < 0 || atlasRows > 32768) return arg_error(fn, "atlasRows must be in [0, 32768]");
  if (atlasWidth < 1 || atlasWidth > 32768) return arg_error(fn, "atlasWidth must be in [1, 32768]");
  if (padding < 0 || padding > 16) return arg_error(fn, "padding must be in [0, 16]");
  if (!local && (!std::isfinite(smoothness) || smoothness < 0.0))
    return arg_error(fn, "smoothness must be finite and >= 0");
  if (!local && (!std::isfinite(regularization) || regularization <= 0.0))
    return arg_error(fn, "regularization must be finite and > 0");
  if (local && (stripWidth < 1 || stripWidth > 128)) return arg_error(fn, "stripWidth must be in [1, 128]");
  if (maxIterations < 0 || maxIterations > 100000) return arg_error(fn, "maxIterations must be in [0, 100000]");
  if (!(tol >= 0.0 && tol < 1.0)) return arg_error(fn, "tol must be in [0, 1)");
  if (numCharts < 0) return arg_error(fn, "numCharts must be >= 0");
  if (numCharts > 0 && !charts) return arg_error(fn, "numCharts > 0 needs charts");
  for (int c = 0; c < numCharts; c++) {
    const int *e = charts + 8 * (size_t)c;
    if (e[0] < 0 || e[3] < 1 || e[4] < 1 || e[5] < 0 || e[6] < 0 || e[3] > atlasWidth - e[5] ||
        e[4] > atlasRows - e[6])
      return arg_error(fn, "charts[%d] must have an image >= 0 and a rectangle of at least one texel inside the atlas",
                       c);
  }
  // No two chart rectangles may share a texel: a texel belongs to one image, and rule 1 finds a face's chart by one
  // search of the row index.  A sweep over x (a chart leaves at ox + width before any chart enters there) keeps the
  // charts that cover the current column by oy; they are disjoint in y, so a chart entering overlaps one of them
  // exactly when it overlaps its neighbour below or above in oy.
  {
    std::vector<std::array<int, 3>> events;   // (x, enters, chart)
    events.reserve((size_t)2 * numCharts);
    for (int c = 0; c < numCharts; c++) {
      const int *e = charts + 8 * (size_t)c;
      events.push_back({e[5] + e[3], 0, c});
      events.push_back({e[5], 1, c});
    }
    std::sort(events.begin(), events.end());
    std::set<std::pair<int, int>> active;     // (oy, chart)
    for (const auto &ev : events) {
      const int c = ev[2], oy = charts[8 * (size_t)c + 6], h = charts[8 * (size_t)c + 4];
      if (!ev[1]) {
        active.erase({oy, c});
        continue;
      }
      auto above = active.lower_bound({oy, -1});
      int other = -1;
      if (above != active.end() && above->first < oy + h) other = above->second;
      if (other < 0 && above != active.begin()) {
        const auto below = std::prev(above);
        if (below->first + charts[8 * (size_t)below->second + 4] > oy) other = below->second;
      }
      if (other >= 0)
        return arg_error(fn, "charts[%d] and charts[%d] must not overlap", std::min(c, other), std::max(c, other));
      active.insert({oy, c});
    }
  }
  if (numVertices > 0 && (!vertices || misaligned(vertices, 4)))
    return arg_error(fn, "numVertices > 0 needs d_vertices (4-byte aligned)");
  if (numTriangles > 0 && (!triangles || misaligned(triangles, 4)))
    return arg_error(fn, "numTriangles > 0 needs d_triangles (4-byte aligned)");
  if (numTriangles > 0 && (!faceView || misaligned(faceView, 4)))
    return arg_error(fn, "numTriangles > 0 needs d_faceView (4-byte aligned)");
  if (numTriangles > 0 && (!uv || misaligned(uv, 4)))
    return arg_error(fn, "numTriangles > 0 needs d_uv (4-byte aligned)");
  if (!local && numTriangles > 0 && (!cornerOffset || misaligned(cornerOffset, 4)))
    return arg_error(fn, "numTriangles > 0 needs d_cornerOffset (4-byte aligned)");
  const size_t texels = (size_t)atlasRows * atlasWidth;
  if (texels > 0 && (!atlas || misaligned(atlas, 4))) return arg_error(fn, "atlasRows > 0 needs d_atlas (4-byte aligned)");
  if (texels > 0 && (!outAtlas || misaligned(outAtlas, 4)))
    return arg_error(fn, "atlasRows > 0 needs d_outAtlas (4-byte aligned)");
  // the outputs (written), the mesh, the labels, the coordinates and the atlas (read)
  static const char *const names[7] = {"d_outAtlas", "d_cornerOffset", "d_vertices", "d_triangles",
                                       "d_faceView", "d_uv", "d_atlas"};
  ArgRanges rs(names, 7);
  const size_t T = (size_t)numTriangles;
  rs.add(outAtlas, 4 * texels, 0, 0, true);
  if (!local) rs.add(cornerOffset, 12 * T, 1, 0, true);
  rs.add(vertices, 12 * (size_t)numVertices, 2, 0, false);
  rs.add(triangles, 12 * T, 3, 0, false);
  rs.add(faceView, 4 * T, 4, 0, false);
  rs.add(uv, 24 * T, 5, 0, false);
  rs.add(atlas, 4 * texels, 6, 0, false);
  return rs.check(fn);
}

}  // namespace cs
