"""Randomised checks of the buffer-overlap rule of every C ABI call that takes device buffers.  Each layout places the
call's buffers at random 8-byte aligned offsets in one host arena and holds at least one forbidden overlap, so no call
can reach a device.  The call must return CS_E_ARG, the two ranges its message names must share a byte and may not
share one under the call's rule (restated here pairwise), and no byte of the arena may be written."""
import ctypes
import re

import numpy as np
import pytest

import cudasift_b200 as cs

CS_E_ARG = -2
REC = 576
LAYOUTS = 300
K = np.array([[800.0, 0, 640], [0, 800, 480], [0, 0, 1]])
H = np.eye(3)
MSG = re.compile(r"^[^:]+(?:: (jobs\[\d+\]))?: invalid argument \(CS_E_ARG\): (\S+) and (\S+) overlap$")

_buf = np.zeros(1 << 20, np.uint8)
BASE = _buf.ctypes.data + (-_buf.ctypes.data) % 64


def exclusive(names):
    """The rule of most calls: a range named in `names` may share no byte with any other range."""
    return lambda a, b: a in names or b in names


def _job(name):
    return name.split(".")[0]


def _counts(rng, k, lo=1, hi=5):
    return [int(v) for v in rng.integers(lo, hi, k)]


# Each layout function returns (sizes, forbidden, call): sizes maps a range's name (as the library names it) to its
# bytes, forbidden(a, b) says whether ranges a and b may not share a byte, and call(at) makes the call with range x at
# address at[x].


def single(rng, fn, sets_written=False):
    n1, n2, np_, ni = _counts(rng, 4)
    L = cs.lib()
    ms = ctypes.c_double()
    model = np.zeros(12)
    d = model.ctypes.data
    if fn in ("cs_match_knn2", "cs_match_knn2_guided"):
        sizes = dict(idx=8 * n1, score=8 * n1)
    elif fn in ("cs_verify_pairs", "cs_verify_pairs_host", "cs_verify_essential", "cs_verify_essential_host"):
        sizes = dict(pairs=8 * np_, inliers=8 * ni)
    else:
        sizes = dict(pairs=8 * np_)
    excl = set(sizes) | ({"s1", "s2"} if sets_written else set())
    sizes.update(s1=n1 * REC, s2=n2 * REC)

    def call(at):
        s = (at["s1"], n1, at["s2"], n2)
        if fn in ("cs_match_mutual", "cs_match_mutual_host"):
            return getattr(L, fn)(*s, 0.0, 1.0, at["pairs"], np_, 0, ms)
        if fn in ("cs_match_ratio", "cs_match_ratio_host"):
            return getattr(L, fn)(*s, 0.8, 1.0, 1, at["pairs"], np_, 0, ms)
        if fn == "cs_match_knn2":
            return L.cs_match_knn2(*s, at["idx"], at["score"], 0, ms)
        if fn == "cs_match_knn2_guided":
            return L.cs_match_knn2_guided(*s, 1, H.ctypes.data, 4.0, at["idx"], at["score"], ms)
        if fn in ("cs_match_guided", "cs_match_guided_host"):
            return getattr(L, fn)(*s, 1, H.ctypes.data, 4.0, 0.8, 1.0, 1, at["pairs"], np_, ms)
        if fn in ("cs_verify_pairs", "cs_verify_pairs_host"):
            return getattr(L, fn)(*s, at["pairs"], np_, 2, 64, 1.0, 1, d, at["inliers"], ni, ms)
        if fn == "cs_verify_models":
            return L.cs_verify_models(*s, at["pairs"], np_, 2, 64, 1.0, 1, d, d, d)
        if fn in ("cs_verify_essential", "cs_verify_essential_host"):
            return getattr(L, fn)(*s, at["pairs"], np_, K.ctypes.data, K.ctypes.data, 64, 1.0, 1, d, d, d,
                                  at["inliers"], ni, ms)
        assert fn == "cs_verify_essential_models", fn
        return L.cs_verify_essential_models(*s, at["pairs"], np_, K.ctypes.data, K.ctypes.data, 64, 1.0, 1, d, d, d)

    return sizes, exclusive(excl), call


def verify_batch(rng, essential):
    J = int(rng.integers(2, 6))
    jobs = [dict(n1=n1, n2=n2, np=p, ni=i) for n1, n2, p, i in zip(*[_counts(rng, J) for _ in range(4)])]
    sizes = {}
    for p, j in enumerate(jobs):
        sizes.update({"jobs[%d].s1" % p: j["n1"] * REC, "jobs[%d].s2" % p: j["n2"] * REC,
                      "jobs[%d].pairs" % p: 8 * j["np"], "jobs[%d].inliers" % p: 8 * j["ni"]})

    def forbidden(a, b):   # an inlier buffer against anything; within a job, the pairs as well
        return a.endswith(".inliers") or b.endswith(".inliers") or (
            _job(a) == _job(b) and (a.endswith(".pairs") or b.endswith(".pairs")))

    out = np.zeros(J * 10)
    Ks = np.stack([K] * J)

    def call(at):
        t = (cs.VerifyJob * J)(*[cs.VerifyJob(at["jobs[%d].s1" % p], j["n1"], at["jobs[%d].s2" % p], j["n2"],
                                              at["jobs[%d].pairs" % p], j["np"], p, at["jobs[%d].inliers" % p], j["ni"])
                                 for p, j in enumerate(jobs)])
        c, o = np.zeros(J, np.int32), out.ctypes.data
        if essential:
            return cs.lib().cs_verify_essential_batch(t, J, Ks.ctypes.data, Ks.ctypes.data, 64, 1.0, o, o, o,
                                                      c.ctypes.data, None, None)
        return cs.lib().cs_verify_pairs_batch(t, J, 2, 64, 1.0, o, c.ctypes.data, None, None)

    return sizes, forbidden, call


def match_batch(rng, guided):
    S, J = (int(v) for v in rng.integers(1, 6, 2))
    n, mp = _counts(rng, S), _counts(rng, J)
    pair = rng.integers(0, S, (J, 2))
    sizes = {"sets[%d].pts" % s: n[s] * REC for s in range(S)}
    sizes.update({"jobs[%d].pairs" % p: 8 * mp[p] for p in range(J)})
    models, Hs = np.ones(J, np.int32), np.stack([H] * J)

    def call(at):
        st = (cs.MatchSet * S)(*[cs.MatchSet(at["sets[%d].pts" % s], n[s]) for s in range(S)])
        jt = (cs.MatchJob * J)(*[cs.MatchJob(int(pair[p, 0]), int(pair[p, 1]), at["jobs[%d].pairs" % p], mp[p])
                                 for p in range(J)])
        c = np.zeros(J, np.int32)
        if guided:
            return cs.lib().cs_match_guided_batch(st, S, jt, J, models.ctypes.data, Hs.ctypes.data, 4.0, 0.8, 1.0, 1,
                                                  c.ctypes.data, None, None)
        return cs.lib().cs_match_ratio_batch(st, S, jt, J, 0.8, 1.0, 1, c.ctypes.data, None, None)

    return sizes, exclusive({"jobs[%d].pairs" % p for p in range(J)}), call


def tracks(rng):
    I, Lc = (int(v) for v in rng.integers(1, 5, 2))
    imageSizes = np.array(_counts(rng, I, 1, 9), np.int32)
    npairs, img = _counts(rng, Lc), rng.integers(0, I, (Lc, 2))
    maxTracks, maxMembers = _counts(rng, 2)
    outs = dict(d_trackOf=4 * int(imageSizes.sum()), d_offsets=4 * (maxTracks + 1), d_members=8 * maxMembers)
    sizes = dict(outs, **{"lists[%d].pairs" % p: 8 * npairs[p] for p in range(Lc)})

    def call(at):
        lt = (cs.TrackList * Lc)(*[cs.TrackList(int(img[p, 0]), int(img[p, 1]), at["lists[%d].pairs" % p], npairs[p])
                                   for p in range(Lc)])
        return cs.lib().cs_build_tracks(imageSizes.ctypes.data, I, lt, Lc, 2, 1, at["d_trackOf"], at["d_offsets"],
                                        maxTracks, at["d_members"], maxMembers, None, None)

    return sizes, exclusive(set(outs)), call


def cameras(rng):
    I = int(rng.integers(1, 4))
    n = _counts(rng, I)
    Ks, Rs, ts = np.stack([K] * I), np.stack([np.eye(3)] * I), np.zeros((I, 3))
    sizes = {"sets[%d].pts" % a: n[a] * REC for a in range(I)}
    return I, n, (Ks, Rs, ts), sizes


def triangulate(rng):
    I, n, cam, sizes = cameras(rng)
    T, M = _counts(rng, 2)
    outs = dict(d_points=24 * T, d_counts=4 * T, d_errors=4 * M, d_inlier=M)
    sizes.update(outs, d_offsets=4 * (T + 1), d_members=8 * M)

    def call(at):
        st = (cs.MatchSet * I)(*[cs.MatchSet(at["sets[%d].pts" % a], n[a]) for a in range(I)])
        return cs.lib().cs_triangulate_tracks(st, I, *(x.ctypes.data for x in cam), at["d_offsets"], T,
                                              at["d_members"], M, 64, 4.0, 1.0, 1, at["d_points"], at["d_counts"],
                                              at["d_errors"], at["d_inlier"], None, None)

    return sizes, exclusive(set(outs)), call


def bundle(rng):
    I, n, cam, sizes = cameras(rng)
    T, M = _counts(rng, 2)
    outs = dict(d_points=24 * T, d_errors=4 * M, d_inlier=M)
    sizes.update(outs, d_offsets=4 * (T + 1), d_members=8 * M, d_use=M)
    R, t, cost = np.zeros((I, 9)), np.zeros((I, 3)), np.zeros(2)

    def call(at):
        st = (cs.MatchSet * I)(*[cs.MatchSet(at["sets[%d].pts" % a], n[a]) for a in range(I)])
        return cs.lib().cs_bundle_adjust(st, I, *(x.ctypes.data for x in cam), None, at["d_offsets"], T,
                                         at["d_members"], M, at["d_use"], at["d_points"], 10, 50, 0.1, 4.0,
                                         R.ctypes.data, t.ctypes.data, at["d_errors"], at["d_inlier"], cost.ctypes.data,
                                         None, None, None)

    return sizes, exclusive(set(outs)), call


def pose(rng, models):
    J = 1 if models else int(rng.integers(1, 5))
    n, P = _counts(rng, J), int(rng.integers(1, 5))
    sizes = {"d_points": 24 * P}
    for p in range(J):
        sizes.update({"jobs[%d].pts" % p: n[p] * REC, "jobs[%d].pointOf" % p: 4 * n[p],
                      "jobs[%d].errors" % p: 4 * n[p], "jobs[%d].inlier" % p: n[p]})
    Ks = np.stack([K] * J)
    out = np.zeros(J * 9 * 64)

    def call(at):
        t = (cs.PoseJob * J)(*[cs.PoseJob(at["jobs[%d].pts" % p], n[p], at["jobs[%d].pointOf" % p], p,
                                          at["jobs[%d].errors" % p], at["jobs[%d].inlier" % p]) for p in range(J)])
        o = out.ctypes.data
        if models:
            return cs.lib().cs_absolute_pose_models(at["d_points"], P, t, Ks.ctypes.data, 64, 4.0, o, o, o)
        return cs.lib().cs_absolute_pose_batch(at["d_points"], P, t, J, Ks.ctypes.data, 64, 4.0, o, o, o, None, None)

    return sizes, lambda a, b: a.endswith((".errors", ".inlier")) or b.endswith((".errors", ".inlier")), call


SINGLE = ["cs_match_ratio", "cs_match_ratio_host", "cs_match_knn2", "cs_match_knn2_guided", "cs_match_guided",
          "cs_match_guided_host", "cs_verify_pairs", "cs_verify_pairs_host", "cs_verify_models", "cs_verify_essential",
          "cs_verify_essential_host", "cs_verify_essential_models"]
CALLS = dict({fn: (lambda fn: lambda rng: single(rng, fn))(fn) for fn in SINGLE}, **{
    "cs_match_mutual": lambda rng: single(rng, "cs_match_mutual", sets_written=True),
    "cs_match_mutual_host": lambda rng: single(rng, "cs_match_mutual_host", sets_written=True),
    "cs_verify_pairs_batch": lambda rng: verify_batch(rng, False),
    "cs_verify_essential_batch": lambda rng: verify_batch(rng, True),
    "cs_match_ratio_batch": lambda rng: match_batch(rng, False),
    "cs_match_guided_batch": lambda rng: match_batch(rng, True),
    "cs_build_tracks": tracks,
    "cs_triangulate_tracks": triangulate,
    "cs_bundle_adjust": bundle,
    "cs_absolute_pose_batch": lambda rng: pose(rng, False),
    "cs_absolute_pose_models": lambda rng: pose(rng, True),
})


def _share(x, y):
    return x[0] < y[0] + y[1] and y[0] < x[0] + x[1]


def _layout(rng, sizes, forbidden):
    """Random 8-byte aligned offsets with at least one forbidden overlap (one range moved onto another when the draw
    has none)."""
    names = sorted(sizes)
    span = max(8, int(sum(sizes.values()) * rng.uniform(0.5, 2.0)) // 8 * 8)
    at = {x: 8 * int(rng.integers(0, span // 8)) for x in names}
    bad = [(a, b) for a in names for b in names if a < b and forbidden(a, b)]
    assert bad
    if not any(_share((at[a], sizes[a]), (at[b], sizes[b])) for a, b in bad):
        a, b = bad[int(rng.integers(0, len(bad)))]
        at[a] = at[b] + 8 * int(rng.integers(0, (sizes[b] - 1) // 8 + 1))
    return at


@pytest.mark.parametrize("fn", sorted(CALLS))
def test_every_overlap_is_rejected_and_named(fn):
    rng = np.random.default_rng(sum(map(ord, fn)))
    for _ in range(LAYOUTS):
        sizes, forbidden, call = CALLS[fn](rng)
        at = _layout(rng, sizes, forbidden)
        assert max(at[x] + sizes[x] for x in sizes) <= _buf.size - 64
        r = call({x: BASE + v for x, v in at.items()})
        msg = cs.lib().cs_last_error().decode()
        assert r == CS_E_ARG, (fn, r, msg, at, sizes)
        m = MSG.match(msg)
        assert m, (fn, msg)
        job, a, b = m.groups()
        if job:                                                 # a batch job checked as its single call
            a, b = job + "." + a, job + "." + b
        assert a in sizes and b in sizes, (fn, msg, sorted(sizes))
        assert forbidden(a, b) and _share((at[a], sizes[a]), (at[b], sizes[b])), (fn, msg, at, sizes)
    assert not _buf.any(), fn
