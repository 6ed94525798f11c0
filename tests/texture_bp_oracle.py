"""cs_texture_mesh_bp's rule 4b restated in float64 (numpy element-wise operations, each rounded once, in the header's
order): the min-sum messages over the Potts factors, a colour step at a time, the decode, the energy of every decoded
labelling and the keep rule.  Rules 1 to 3c, 4a, 5 and 6 are texture_photo_oracle.texture_photo's, unchanged: for the
length of a call texture_oracle's `energy` stands for "E of the start labelling, then BP" on its first use, and hands
the ICM sweeps the kept labelling in place; `colouring` is watched for the colours."""
import numpy as np

import texture_oracle as to
import texture_photo_oracle as tpo

MCAND = to.MCAND
INF = np.inf


def data_terms(cands):
    """D [T, MCAND] (+inf past a face's count), the images A [T, MCAND] (-1 past it) and the counts m [T]."""
    T = len(cands)
    D, A, m = np.full((T, MCAND), INF), np.full((T, MCAND), -1, np.int64), np.zeros(T, np.int64)
    for f, c in enumerate(cands):
        m[f] = len(c)
        for r, (q, a) in enumerate(c):
            D[f, r] = 1.0 - q / c[0][0]
            A[f, r] = a
    return D, A, m


def factors(tris, nbr, m):
    """Per slot (f, k) with seen f and seen g across it: g's slot k' with the same two vertex ids (-1 elsewhere)."""
    t = np.asarray(tris, np.int64)
    T = len(t)
    kp = np.full((T, 3), -1, np.int64)
    for f in range(T):
        if m[f] == 0:
            continue
        for k in range(3):
            g = nbr[f, k]
            if g < 0 or m[g] == 0:
                continue
            e = {t[f, k], t[f, (k + 1) % 3]}
            kp[f, k] = [j for j in range(3) if {t[g, j], t[g, (j + 1) % 3]} == e][0]
    return kp


def rank_map(A, f, g):
    """R [n, MCAND]: for each of g's ranks r', the rank of the same image among f's candidates (-1 when absent)."""
    same = A[f][:, :, None] == A[g][:, None, :]
    same &= A[f][:, :, None] >= 0
    return np.where(same.any(1), same.argmax(1), -1)


def excluded(D, msg, F, k):
    """h [n, MCAND]: D(f, r) + the messages into f at the slots j != k, added in ascending j."""
    h = D[F].copy()
    for j in range(3):
        if j != k:
            h = h + msg[F, j]
    return h


def normalise(M, mg):
    """The message: M minus its minimum over g's ranks; entries past g's count are 0."""
    valid = np.arange(MCAND)[None, :] < mg[:, None]
    lo = np.where(valid, M, INF).min(1)
    return np.where(valid, M - lo[:, None], 0.0)


def colour_step(D, A, m, nbr, kp, msg, col, c, lam):
    """Every message out of every seen face of colour c; returns the number of messages that changed a bit."""
    changed = 0
    F0 = np.nonzero((col == c) & (m > 0))[0]
    for k in range(3):
        F = F0[kp[F0, k] >= 0]
        if not len(F):
            continue
        G, K = nbr[F, k], kp[F, k]
        h = excluded(D, msg, F, k)
        hmin = h.min(1)
        R = rank_map(A, F, G)
        hr = np.where(R >= 0, np.take_along_axis(h, np.maximum(R, 0), 1), INF)
        M = np.minimum(hr, (hmin + lam)[:, None])
        new = normalise(M, m[G])
        old = msg[G, K]
        changed += int((new.view(np.uint64) != old.view(np.uint64)).any(1).sum())
        msg[G, K] = new
    return changed


def decode(D, A, m, msg):
    """The labels: a_f[r*], r* the lowest rank of minimum D + every message into f in ascending slot order."""
    b = ((D + msg[:, 0]) + msg[:, 1]) + msg[:, 2]
    r = b.argmin(1)
    lab = np.where(m > 0, A[np.arange(len(m)), r], -1)
    return lab, r


def energy(label, D, A, nbr, lam):
    """Rule 4's E, vectorised: e_f = D(f, l_f) + lambda #{g > f across an edge, labelled, l_g != l_f}."""
    T = len(label)
    seen = label >= 0
    r = (A == label[:, None]).argmax(1)
    Dl = D[np.arange(T), r]
    g = nbr
    lg = np.where(g >= 0, label[np.maximum(g, 0)], -1)
    dis = ((g > np.arange(T)[:, None]) & (lg >= 0) & (lg != label[:, None])).sum(1)
    e = np.where(seen, Dl + lam * dis.astype(np.float64), 0.0)
    return to.tree_total(e)


def step(D, A, m, nbr, kp, msg, col, colours, lam):
    """One sweep: colours 0, 1, ... in order.  Returns the messages changed."""
    return sum(colour_step(D, A, m, nbr, kp, msg, col, c, lam) for c in range(colours))


def keep(e, best):
    return e < best


def converged(changed, moved_labels):
    return changed == 0


def belief_propagation(label, e0, cands, nbr, tris, col, lam, maxBpSweeps):
    """Rule 4b from the start labelling, whose E is e0 (label changed in place to the kept labelling).  Returns
    (E_kept, stats [16..19])."""
    D, A, m = data_terms(cands)
    if maxBpSweeps == 0:
        return e0, [0, 0, 0, 0]
    kp = factors(tris, nbr, m)
    colours = int(col.max()) + 1
    msg = np.zeros((len(label), 3, MCAND))
    kept, ek, sweep, kept_at, last, moved = label.copy(), e0, 0, 0, 0, 0
    prev = label.copy()
    while sweep < maxBpSweeps:
        last = step(D, A, m, nbr, kp, msg, col, colours, lam)
        lab, r = decode(D, A, m, msg)
        sweep += 1
        e = energy(lab, D, A, nbr, lam)
        if keep(e, ek):
            kept, ek, kept_at, moved = lab, e, sweep, int(((r != 0) & (m > 0)).sum())
        if converged(last, not np.array_equal(lab, prev)):
            break
        prev = lab
    label[:] = kept
    return ek, [sweep, kept_at, last, moved]


def polish(after, kept):
    """The labels the charts use: those after the ICM sweeps from the kept labelling (a hook for the mutations)."""
    return after


def texture_bp(images, Ks, Rs, ts, verts, tris, maxBpSweeps=32, **kw):
    """The whole call: texture_photo_oracle.texture_photo's dict with info [3] and stats [20]."""
    rule_energy, rule_colouring = to.energy, to.colouring
    state = {}

    def colouring(nbr):
        col, rounds = rule_colouring(nbr)
        state["col"] = col
        return col, rounds

    def energy_hook(label, cands, nbr, lam):
        if "bp" in state:
            label[:] = polish(label.copy(), state["kept"])
            return rule_energy(label, cands, nbr, lam)
        e0 = rule_energy(label, cands, nbr, lam)
        ek, st = belief_propagation(label, e0, cands, nbr, tris, state["col"], lam, maxBpSweeps)
        state["bp"], state["kept"] = (ek, st), label.copy()
        return e0

    to.energy, to.colouring = energy_hook, colouring
    try:
        r = tpo.texture_photo(images, Ks, Rs, ts, verts, tris, **kw)
    finally:
        to.energy, to.colouring = rule_energy, rule_colouring
    ek, st = state.get("bp", (0.0, [0, 0, 0, 0]))
    r["info"] = list(r["info"]) + [ek]
    r["stats"] = list(r["stats"]) + st
    r["kept"] = state.get("kept")
    return r
