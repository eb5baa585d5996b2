"""CPU restatement of continuous collision (nb_upload_ccd_bodies; k_ccd and k_advance<true> in nudge_b200/csrc) by brute force over every
collider — TEST INFRASTRUCTURE ONLY.

The reference has no continuous collision.  This follows the float32 arithmetic include/nudge_b200.h states, operation by operation (numpy
float32 ufuncs round every operation and never fuse), vectorised over every (entry, candidate collider) pair of one step.  The per-collider
tests are the shape casts' and overlap queries' restatements, reused: overlap_ref's step-0 sphere tests, shapecast_ref.rounded_box for a
box and raycast_ref._sphere with the summed radius for a sphere.  What is new here is which colliders count: the body's own, sensors,
colliders failing Box2D's rule against the entry's (category, mask), colliders of a connected body (when asked) and, unlike nb_shapecast,
colliders the sphere touches at its start are skipped; and which entries cast: advanced bodies whose translation is longer than their
threshold.  A touch at t = 0 that is not a start counts only when the motion points into the collider (dot of the step-0 test's gap and the
motion), so that a sphere clamped onto a face, where the face slab and step 0 can round its start apart, still moves away or along the
face.  The colliders, their world transforms and sensor flags are raycast_ref.Scene's.  Before the exact arithmetic shapecast_ref's float64
reach test drops the colliders each swept sphere cannot reach; whether and where a collider is hit is decided by the exact arithmetic alone."""
import numpy as np
from nudge_b200 import abi
from oracle.joints_ref import qrot, dot
from oracle import overlap_ref, raycast_ref, shapecast_ref
from oracle.raycast_ref import Scene  # noqa: F401  (continuous collision's scene too)

f = np.float32
NO_HIT = abi.RAY_NO_HIT
FILTER_ALL = 0xffffffff


def filter_words(filters, k):
    """The colliders' filter words category | mask << 16 (scenes.FILTER rows), NB_FILTER_ALL for each without a table."""
    if filters is None:
        return np.full(k, FILTER_ALL, np.uint64)
    return np.asarray(filters["category"], np.uint64) | (np.asarray(filters["mask"], np.uint64) << np.uint64(16))


def _pass(wa, wb):
    """Box2D's rule on filter words (k_grid_pairs' filter_pass)."""
    return ((wa & (wb >> np.uint64(16))) != 0) & ((wb & (wa >> np.uint64(16))) != 0)


def cast(scene, entries, p, d, filters=None, connected=(), start_skip=True):
    """(t, collider) per entry of abi.CCD_BODY rows `entries`: its sphere cast from p[k] along d[k] with max_t = 1 against the counted
    colliders, t = 1.0 and collider = NO_HIT without a hit.  connected: pairs (a, b) of connected bodies whose colliders the body skips (the
    NB_FILTER_SKIP_CONNECTED lookup; empty without the flag).  start_skip=False makes a collider touched at the start a t = 0 hit, as in
    nb_shapecast."""
    entries = np.asarray(entries, abi.CCD_BODY).reshape(-1)
    n, S = len(entries), scene
    t_out, c_out = np.ones(n, f), np.full(n, NO_HIT, np.uint32)
    k = len(S.body)
    if not n or not k:
        return t_out, c_out
    p, d = np.asarray(p, f).reshape(n, 3), np.asarray(d, f).reshape(n, 3)
    r = entries["radius"].astype(f)
    body = entries["body"].astype(np.int64)
    words = filter_words(filters, k)
    ew = entries["category"].astype(np.uint64) | (entries["mask"].astype(np.uint64) << np.uint64(16))
    conn = {(min(a, b), max(a, b)) for a, b in connected}
    # candidates: shapecast_ref's float64 reach test of each entry's swept sphere.  Its reach is at most A + (|w| + rr) / 256 with |w| at most
    # the distance to the segment's midpoint plus |d| / 2, which bounds that distance first (one matrix product per chunk of entries); the
    # few colliders within the bound get the test itself.
    P64, rad = S.p64, S.radius64
    big = 1.0 + 2.0 * float(np.abs(P64).max()) + float(np.abs(p).max())
    pn = (P64 * P64).sum(axis=1)
    pe, ce = [], []
    for e0 in range(0, n, 128):
        c64, d64, r64 = p[e0:e0 + 128].astype(np.float64), d[e0:e0 + 128].astype(np.float64), r[e0:e0 + 128].astype(np.float64)
        mid, half = c64 + 0.5 * d64, 0.5 * np.linalg.norm(d64, axis=1)
        k = 1 + 2.0 ** -6 + 2.0 ** -8 + 1e-4   # A = k rr + 1e-4 big, rr = r + the collider's radius: the bound splits into two sums
        be = (half * (1 + 2.0 ** -8) + k * r64 + 1e-4 * big) / (1 - 2.0 ** -8) + 1e-6 * big
        bound = be[:, None] + (k / (1 - 2.0 ** -8)) * rad[None, :]
        dist2 = pn[None, :] - 2.0 * (mid @ P64.T)
        dist2 += (mid * mid).sum(axis=1)[:, None]
        bound *= bound
        ee, ii = np.nonzero(dist2 <= bound)
        w = P64[ii] - c64[ee]
        dv = d64[ee]
        tp = np.clip((w * dv).sum(axis=1) / np.maximum((dv * dv).sum(axis=1), 1e-300), 0.0, 1.0)
        dist = np.linalg.norm(w - tp[:, None] * dv, axis=1)
        rr = r64[ee] + rad[ii]
        reach = rr * (1 + 2.0 ** -6) + 1e-4 * (1.0 + np.abs(c64[ee]).max(axis=1) + 2.0 * np.abs(P64[ii]).max(axis=1) + rr) + \
            (np.linalg.norm(w, axis=1) + rr) / 256.0
        keep = dist <= reach
        pe.append(ee[keep] + e0); ce.append(ii[keep])
    e_of, i_of = np.concatenate(pe), np.concatenate(ce)
    ok = (S.body[i_of].astype(np.int64) != body[e_of]) & ~S.sensor[i_of] & _pass(ew[e_of], words[i_of])
    if conn:
        ok &= np.array([(min(a, b), max(a, b)) not in conn for a, b in zip(body[e_of], S.body[i_of].astype(np.int64))], bool)
    e_of, i_of = e_of[ok], i_of[ok]
    m = len(i_of)
    if not m:
        return t_out, c_out
    P, Q, H = S.world["position"][i_of], S.world["rotation"][i_of], S.half[i_of]
    c = tuple(p[e_of, a] for a in range(3))
    dd = tuple(d[e_of, a] for a in range(3))
    rr = r[e_of]
    isbox = i_of < S.nboxes
    start, hit, t = np.zeros(m, bool), np.zeros(m, bool), np.zeros(m, f)
    with np.errstate(all="ignore"):
        b = isbox
        if b.any():
            Pb, Qb, Hb = tuple(P[b, a] for a in range(3)), tuple(Q[b, a] for a in range(4)), tuple(H[b, a] for a in range(3))
            cb = tuple(x[b] for x in c)
            start[b] = overlap_ref._sphere_box(cb, rr[b], Pb, Qb, Hb)
            qc = (-Qb[0], -Qb[1], -Qb[2], Qb[3])
            lo = qrot(qc, (cb[0] - Pb[0], cb[1] - Pb[1], cb[2] - Pb[2]))
            ld = qrot(qc, tuple(x[b] for x in dd))
            hit[b], t[b], _ = shapecast_ref.rounded_box(lo, ld, Hb, rr[b], f(1.0))
        s = ~isbox
        if s.any():
            cs = tuple(x[s] for x in c)
            start[s] = overlap_ref._sphere_sphere(cs, rr[s], tuple(P[s, a] for a in range(3)), H[s, 0])
            hit[s], t[s], _ = raycast_ref._sphere(cs, tuple(x[s] for x in dd), f(1.0), P[s], rr[s] + H[s, 0])
    if start_skip:   # a start is skipped, and another touch at t = 0 counts only when d points into the collider
        into = np.zeros(m, bool)
        if b.any():
            into[b] = dot(tuple(overlap_ref._gap(lo[k], Hb[k]) for k in range(3)), ld) < 0
        if s.any():
            into[s] = dot(tuple(c[k][s] - P[s, k] for k in range(3)), tuple(x[s] for x in dd)) < 0
        hit &= ~start & ((t != 0) | into)
    else:
        hit |= start
        t = np.where(start, f(0.0), t)
    keys = (t.view(np.uint32).astype(np.uint64) << np.uint64(32)) | i_of.astype(np.uint64)
    keys[~hit] = np.uint64(0xffffffffffffffff)
    best = np.full(n, np.uint64(0xffffffffffffffff))
    np.minimum.at(best, e_of, keys)
    got = best != np.uint64(0xffffffffffffffff)
    t_out[got] = (best[got] >> np.uint64(32)).astype(np.uint32).view(f)
    c_out[got] = (best[got] & np.uint64(0xffffffff)).astype(np.uint32)
    return t_out, c_out


def valid(d):
    """Whether each translation is a valid sweep direction with max_t = 1 (finite, not zero)."""
    return np.isfinite(d).all(axis=1) & (d != 0).any(axis=1)


def step(scene, entries, p, v, dt, advanced, filters=None, connected=()):
    """One nb_advance of the set: (t, collider, position) per entry.  p = the bodies' positions as nb_advance finds them, v = their
    velocities after the solver (rows per entry), advanced = whether the step advances each entry's body (awake, not kinematic).  An entry
    casts when advanced, (d.x*d.x + d.y*d.y) + d.z*d.z > threshold * threshold and d is valid, d = v * dt per axis; position = p + d * t per
    axis (t = 1 without a hit: p + d), and p for a body the step does not advance."""
    entries = np.asarray(entries, abi.CCD_BODY).reshape(-1)
    p, v = np.asarray(p, f).reshape(-1, 3), np.asarray(v, f).reshape(-1, 3)
    d = v * f(dt)
    thr = entries["motion_threshold"].astype(f)
    with np.errstate(all="ignore"):
        go = np.asarray(advanced, bool) & (((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]) > thr * thr) & valid(d)
    t, col = np.ones(len(entries), f), np.full(len(entries), NO_HIT, np.uint32)
    if go.any():
        t[go], col[go] = cast(scene, entries[go], p[go], d[go], filters, connected)
    return t, col, np.where(np.asarray(advanced, bool)[:, None], p + d * t[:, None], p)
