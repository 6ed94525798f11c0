"""A numpy statement of cs_build_tracks (include/cudasift_b200.h), to read against the header.

Global ids: feature f of image a is g = base[a] + f with base the exclusive prefix of the image sizes.  Components come
from union-find over the global ids: every round hooks the larger root of each pair that joins two trees onto the
smaller one (the smallest candidate wins), then points every feature at its root.  A root only ever gets a smaller
parent, so each final root is its component's smallest id.  Then the header's rules follow: matched features, the
order (label, g), the conflict rule, minLength and dropConflicting, truncation and the eight statistics.
"""
import numpy as np


def global_pairs(sizes, lists):
    """The valid pairs of lists [(a, b, pairs int [k, 2])] as global ids (u, v), and the invalid pair count."""
    sizes = np.asarray(sizes, np.int64)
    base = np.concatenate([[0], np.cumsum(sizes)])[:-1]
    us, vs, invalid = [], [], 0
    for a, b, p in lists:
        p = np.asarray(p, np.int64).reshape(-1, 2)
        ok = (p[:, 0] >= 0) & (p[:, 0] < sizes[a]) & (p[:, 1] >= 0) & (p[:, 1] < sizes[b])
        invalid += int((~ok).sum())
        us.append(base[a] + p[ok, 0])
        vs.append(base[b] + p[ok, 1])
    cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.int64)
    return cat(us), cat(vs), invalid


def components(n, u, v):
    """Union-find over n ids and the edges (u, v): the label of every id, its component's smallest id."""
    parent = np.arange(n, dtype=np.int64)
    while True:
        ru, rv = parent[u], parent[v]                   # parent is flat here: these are roots
        cross = ru != rv
        if not cross.any():
            return parent
        hi, lo = np.maximum(ru[cross], rv[cross]), np.minimum(ru[cross], rv[cross])
        np.minimum.at(parent, hi, lo)                   # hook each root onto its smallest candidate
        while True:                                     # pointer jumping until every id points at a root
            nxt = parent[parent]
            if np.array_equal(nxt, parent):
                break
            parent = nxt


def build_tracks(sizes, lists, minLength=2, dropConflicting=True, maxTracks=None, maxMembers=None):
    """cs_build_tracks on host data: (T, offsets int32 [min(T, maxTracks) + 1], members int32 [min(M, maxMembers), 2],
    trackOf int32 [N], stats int64 [8]).  maxTracks / maxMembers None: no truncation."""
    sizes = np.asarray(sizes, np.int64)
    N = int(sizes.sum())
    base = np.concatenate([[0], np.cumsum(sizes)])
    u, v, invalid = global_pairs(sizes, lists)
    label = components(N, u, v)
    matched = np.zeros(N, bool)
    matched[u] = True
    matched[v] = True
    g = np.flatnonzero(matched)                          # ascending global id
    g = g[np.argsort(label[g], kind="stable")]           # then by label: one run per component
    lab = label[g]
    image = np.searchsorted(base, g, side="right") - 1
    head = np.ones(len(g), bool)
    head[1:] = lab[1:] != lab[:-1]
    starts = np.flatnonzero(head)
    size = np.diff(np.concatenate([starts, [len(g)]]))
    same = np.zeros(len(g), bool)
    same[1:] = (~head[1:]) & (image[1:] == image[:-1])   # sorted by g, one image's members are adjacent
    conflict = np.add.reduceat(same.astype(np.int64), starts) > 0 if len(g) else np.zeros(0, bool)
    short = size < minLength
    kept = ~short & ~(conflict & bool(dropConflicting))
    T, M = int(kept.sum()), int(size[kept].sum())
    offsets = np.concatenate([[0], np.cumsum(size[kept])]).astype(np.int32)
    run = np.repeat(np.arange(len(starts)), size)        # the run of every sorted position
    track = np.full(len(starts), -1, np.int64)
    track[kept] = np.arange(T)
    trackOf = np.full(N, -1, np.int32)
    trackOf[g] = track[run]
    sel = kept[run]
    members = np.stack([image[sel], g[sel] - base[image[sel]]], axis=1).astype(np.int32).reshape(-1, 2)
    stats = np.array([len(u), invalid, len(g), len(starts), int((conflict & ~short).sum()), int(short.sum()), T, M],
                     np.int64)
    if maxTracks is not None:
        offsets = offsets[:min(T, maxTracks) + 1]
    if maxMembers is not None:
        members = members[:maxMembers]
    return T, offsets, members, trackOf, stats
