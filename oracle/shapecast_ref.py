"""CPU restatement of nb_shapecast (nudge_b200/csrc/nb_query_api.cuh) by brute force over every collider — TEST INFRASTRUCTURE ONLY.

The reference has no scene queries.  This follows the float32 arithmetic include/nudge_b200.h states for nb_shapecast, operation by
operation (numpy float32 ufuncs round every operation and never fuse), vectorised over the colliders of one cast: step 0 is overlap_ref's
test of the shape at its start, sphere against sphere is raycast_ref's sphere test with the summed radius, and the rounded box and the
swept separating axes are restated here.  The colliders, their world transforms, bodies, tags, categories and sensor flags are
raycast_ref.Scene's.  Before the exact arithmetic a float64 test drops the colliders whose bounding sphere the shape's bounding sphere
cannot reach along the centre path, widened by 2^-6 of the radii (the device margin's relative term), 10^-4 of the magnitudes involved
and 2^-8 of the distances the quadratics see; it is skipped for a BOX cast whose rotation is not of unit length to within 2^-10.  Whether
and where a collider is hit is decided by the exact arithmetic alone."""
import itertools
import numpy as np
from nudge_b200 import abi
from oracle.joints_ref import qrot, cross, dot
from oracle import overlap_ref, raycast_ref
from oracle.raycast_ref import Scene  # noqa: F401  (the shape casts' scene too)

f = np.float32
NO_HIT = abi.RAY_NO_HIT
_E = ((f(1), f(0), f(0)), (f(0), f(1), f(0)), (f(0), f(0), f(1)))


def _cols(a):
    return tuple(a[:, k] for k in range(a.shape[1]))


def _slab(lo, ld, h, max_t):
    """nb_raycast's slab test on a ray in the box's frame: (hit, t, local normal), the normal (0, 0, 0) when no axis was recorded."""
    m = len(lo[0])
    enter, exit_ = np.zeros(m, f), np.full(m, max_t, f)
    axis, s, alive = np.full(m, -1), np.zeros(m, f), np.ones(m, bool)
    for k in range(3):
        z = ld[k] == 0
        alive &= ~(z & ((lo[k] < -h[k]) | (lo[k] > h[k])))
        t1 = (-h[k] - lo[k]) / ld[k]; t2 = (h[k] - lo[k]) / ld[k]
        lt = t1 < t2
        near, far = np.where(lt, t1, t2), np.where(lt, t2, t1)
        up = ~z & (near > enter)
        enter = np.where(up, near, enter); axis = np.where(up, k, axis); s = np.where(up, np.where(lt, f(-1.0), f(1.0)), s)
        exit_ = np.where(~z & (far < exit_), far, exit_)
        alive &= ~(~z & (enter > exit_))
    return alive, enter, [np.where(axis == k, s, f(0.0)) for k in range(3)]


def _root(a, b, cc, max_t):
    disc = b * b - a * cc
    t = (-b - np.sqrt(disc)) / a
    hit = ~(disc < 0) & (t >= 0) & (t <= max_t)
    return hit, np.where(t == 0, f(0.0), t)


def rounded_box(lo, ld, h, r, max_t):
    """A sphere of radius r from lo along ld against the box h centred at the origin, all in the box's frame (per-collider arrays): the
    header's 23 primitives in order, the smallest t winning and the earlier primitive a tie.  Returns (hit, t, local normal)."""
    m = len(r)
    best_hit, best_t, nl = np.zeros(m, bool), np.zeros(m, f), [np.zeros(m, f) for _ in range(3)]

    def take(hit, t, n):
        nonlocal best_hit, best_t
        up = hit & (~best_hit | (t < best_t))
        best_hit = best_hit | up
        best_t = np.where(up, t, best_t)
        for k in range(3):
            nl[k] = np.where(up, n[k], nl[k])

    rp = r != 0
    for k in range(3):   # (a) the face boxes; with r == 0 they are one box
        hit, t, n = _slab(lo, ld, tuple(h[a] + r if a == k else h[a] for a in range(3)), max_t)
        take(hit & (rp if k else True), t, n)
    inv = f(1.0) / r
    for k in range(3):   # (b) the edge cylinders along k
        i, j = [a for a in range(3) if a != k]
        a = ld[i] * ld[i] + ld[j] * ld[j]
        for si, sj in itertools.product((-1.0, 1.0), repeat=2):
            mi, mj = lo[i] - f(si) * h[i], lo[j] - f(sj) * h[j]
            b = mi * ld[i] + mj * ld[j]
            cc = (mi * mi + mj * mj) - r * r
            hit, t = _root(a, b, cc, max_t)
            z = lo[k] + t * ld[k]
            hit &= rp & (a != 0) & (z >= -h[k]) & (z <= h[k])
            n = [None] * 3
            n[i], n[j], n[k] = (mi + t * ld[i]) * inv, (mj + t * ld[j]) * inv, np.zeros(m, f)
            take(hit, t, n)
    a = dot(ld, ld)
    for sg in itertools.product((-1.0, 1.0), repeat=3):   # (c) the corner spheres, x slowest
        c = tuple(f(sg[k]) * h[k] for k in range(3))
        mm = (lo[0] - c[0], lo[1] - c[1], lo[2] - c[2])
        hit, t = _root(a, dot(mm, ld), dot(mm, mm) - r * r, max_t)
        take(hit & rp, t, [((lo[k] + t * ld[k]) - c[k]) * inv for k in range(3)])
    return best_hit, best_t, nl


def _rotated(q, nl, sign=1.0):
    """normal = n_l == (0, 0, 0) ? (0, 0, 0) : sign * qrot(q, n_l), as (m, 3)."""
    w = qrot(q, tuple(nl))
    zero = (nl[0] == 0) & (nl[1] == 0) & (nl[2] == 0)
    return np.stack([np.where(zero, f(0.0), w[k] if sign > 0 else -w[k]) for k in range(3)], axis=1)


def _box_box(c, Qq, H, d, max_t, P, Q, h):
    """The swept separating axes for the query box (c, Qq, H) along d against boxes (P, Q, h): (hit, t, normal)."""
    m = len(P[0])
    one = lambda x: np.full(m, x, f)
    u = [tuple(one(x) for x in qrot(tuple(f(x) for x in Qq), e)) for e in _E]
    v = [qrot(Q, tuple(one(x) for x in e)) for e in _E]
    t0 = (P[0] - c[0], P[1] - c[1], P[2] - c[2])
    Hs, dd = tuple(f(x) for x in H), tuple(one(x) for x in d)

    def radius(hh, ax, L):
        return (np.abs(hh[0] * dot(ax[0], L)) + np.abs(hh[1] * dot(ax[1], L))) + np.abs(hh[2] * dot(ax[2], L))

    enter, exit_, sb = np.zeros(m, f), np.full(m, max_t, f), np.zeros(m, f)
    axis, rec, alive = [np.zeros(m, f) for _ in range(3)], np.zeros(m, bool), np.ones(m, bool)
    for L in u + v + [cross(u[i], v[k]) for i in range(3) for k in range(3)]:
        a, b, R = dot(t0, L), dot(dd, L), radius(Hs, u, L) + radius(h, v, L)
        z = b == 0
        alive &= ~(z & (np.abs(a) > R))
        t1 = (a - R) / b; t2 = (a + R) / b
        lt = t1 < t2
        near, far = np.where(lt, t1, t2), np.where(lt, t2, t1)
        up = ~z & (near > enter)
        enter = np.where(up, near, enter); sb = np.where(up, b, sb); rec |= up
        axis = [np.where(up, L[k], axis[k]) for k in range(3)]
        exit_ = np.where(~z & (far < exit_), far, exit_)
        alive &= ~(~z & (enter > exit_))
    inv = f(1.0) / np.sqrt(dot(axis, axis))
    n = np.stack([np.where(rec, np.where(sb > 0, -axis[k], axis[k]) * inv, f(0.0)) for k in range(3)], axis=1)
    return alive, enter, n


def _valid(cast):
    d, mt = cast["direction"], cast["max_t"]
    return bool(overlap_ref._valid(cast["shape"]) and np.isfinite(d).all() and np.isfinite(mt) and mt >= 0 and (d != 0).any())


def cast(scene, casts, flags=0):
    """abi.RAY_HIT rows for abi.SHAPE_CAST rows, by brute force."""
    casts = np.asarray(casts, abi.SHAPE_CAST).reshape(-1)
    out = np.zeros(len(casts), abi.RAY_HIT)
    out["collider"] = out["body"] = out["tag"] = NO_HIT
    S = scene
    k = len(S.body)
    idx_all = np.arange(k)
    PW, QW = S.world["position"], S.world["rotation"]
    with np.errstate(all="ignore"):
        for n, cs in enumerate(casts):
            if not k or not _valid(cs):
                continue
            q = cs["shape"]
            ok = ((S.category & np.uint32(q["mask"])) != 0) & (S.body != q["ignore_body"])
            if not flags & abi.SHAPECAST_SENSORS:
                ok &= ~S.sensor
            box = int(q["shape"]) == abi.OVERLAP_BOX
            c, d, max_t = tuple(f(x) for x in q["center"]), tuple(f(x) for x in cs["direction"]), f(cs["max_t"])
            # float64 reach test: the collider's bounding sphere against the shape's swept along the centre path [0, max_t], widened
            rot = q["rotation"].astype(np.float64)
            if not (box and abs(float(rot @ rot) - 1.0) > 2.0 ** -10):
                c64, d64 = np.array(c, np.float64), np.array(d, np.float64)
                rq = float(np.linalg.norm(q["half_extents"].astype(np.float64))) if box else float(q["radius"])
                w = S.p64 - c64
                tp = np.clip(w @ d64 / (d64 @ d64), 0.0, float(max_t))
                dist = np.linalg.norm(w - tp[:, None] * d64[None, :], axis=1)
                rr = rq + S.radius64
                ok &= dist <= rr * (1 + 2.0 ** -6) + 1e-4 * (1.0 + np.abs(c64).max() + 2.0 * np.abs(S.p64).max(axis=1) + rr) + \
                    (np.linalg.norm(w, axis=1) + rr) / 256.0
            cand = idx_all[ok]
            if not len(cand):
                continue
            isbox = cand < S.nboxes
            b, s = isbox, ~isbox
            hit, t, nrm = np.zeros(len(cand), bool), np.zeros(len(cand), f), np.zeros((len(cand), 3), f)
            P, Qc, H = PW[cand], QW[cand], S.half[cand]
            start = np.zeros(len(cand), bool)
            if box:
                Qq, Hq = q["rotation"].astype(f), q["half_extents"].astype(f)
                if b.any():
                    start[b] = overlap_ref._box_box(c, Qq, Hq, _cols(P[b]), _cols(Qc[b]), _cols(H[b]))
                    hit[b], t[b], nrm[b] = _box_box(c, Qq, Hq, d, max_t, _cols(P[b]), _cols(Qc[b]), _cols(H[b]))
                if s.any():   # the sphere collider moving along -d against the query box
                    m = int(s.sum())
                    full = lambda x: np.full(m, x, f)
                    Qf, Hf = tuple(full(x) for x in Qq), tuple(full(x) for x in Hq)
                    start[s] = overlap_ref._sphere_box(_cols(P[s]), H[s, 0], tuple(full(x) for x in c), Qf, Hf)
                    qc = (-Qf[0], -Qf[1], -Qf[2], Qf[3])
                    lo = qrot(qc, (P[s, 0] - c[0], P[s, 1] - c[1], P[s, 2] - c[2]))
                    ld = qrot(qc, tuple(full(-x) for x in d))
                    hit[s], t[s], nl = rounded_box(lo, ld, Hf, H[s, 0], max_t)
                    nrm[s] = _rotated(Qf, nl, -1.0)
            else:
                r = f(q["radius"])
                if b.any():
                    Qb, Pb, Hb = _cols(Qc[b]), _cols(P[b]), _cols(H[b])
                    start[b] = overlap_ref._sphere_box(c, r, Pb, Qb, Hb)
                    qc = (-Qb[0], -Qb[1], -Qb[2], Qb[3])
                    lo = qrot(qc, (c[0] - Pb[0], c[1] - Pb[1], c[2] - Pb[2]))
                    ld = qrot(qc, tuple(np.full(len(Pb[0]), x, f) for x in d))
                    hit[b], t[b], nl = rounded_box(lo, ld, Hb, np.full(len(Pb[0]), r, f), max_t)
                    nrm[b] = _rotated(Qb, nl)
                if s.any():
                    start[s] = overlap_ref._sphere_sphere(c, r, _cols(P[s]), H[s, 0])
                    hit[s], t[s], nrm[s] = raycast_ref._sphere(c, d, max_t, P[s], r + H[s, 0])
            hit |= start
            t = np.where(start, f(0.0), t)
            nrm[start] = 0
            if not hit.any():
                continue
            keys = (t.view(np.uint32).astype(np.uint64) << np.uint64(32)) | cand.astype(np.uint64)
            keys[~hit] = np.uint64(0xffffffffffffffff)
            w_ = int(np.argmin(keys))
            tt, i = t[w_], int(cand[w_])
            h = out[n]
            h["t"] = tt
            h["position"] = [c[k] + tt * d[k] for k in range(3)]
            h["normal"] = nrm[w_]
            h["collider"], h["body"], h["tag"] = i, S.body[i], S.tag[i]
    return out
