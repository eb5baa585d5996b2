"""CPU restatement of nb_overlap (nudge_b200/csrc/nb_query_api.cuh) by brute force over every collider — TEST INFRASTRUCTURE ONLY.

The reference has no scene queries.  This follows the float32 arithmetic include/nudge_b200.h states for nb_overlap, operation by
operation (numpy float32 ufuncs round every operation and never fuse), vectorised over the colliders of one query.  The colliders, their
world transforms, bodies, tags, categories and sensor flags are raycast_ref.Scene's.  Before the exact arithmetic a float64 test drops the
colliders whose bounding sphere cannot reach the query's, widened by a relative margin far above float32 rounding; it is skipped for a BOX
query whose rotation is not of unit length to within 2^-10, whose stated test need not stay inside any such sphere.  Whether a collider
overlaps is decided by the exact arithmetic alone."""
import numpy as np
from nudge_b200 import abi
from oracle.joints_ref import qrot, cross, dot
from oracle.raycast_ref import Scene, world_transforms  # noqa: F401  (Scene is the overlap queries' scene too)

f = np.float32
_E = ((f(1), f(0), f(0)), (f(0), f(1), f(0)), (f(0), f(0), f(1)))


def _cols(a):
    return tuple(a[:, k] for k in range(a.shape[1]))


def _gap(l, h):
    return np.where(l < -h, l + h, np.where(l > h, l - h, f(0.0)))


def _sphere_box(c, r, P, Q, H):
    """The sphere (c, r) against boxes (P, Q, H) (c and r may be per box)."""
    qc = (-Q[0], -Q[1], -Q[2], Q[3])
    l = qrot(qc, (c[0] - P[0], c[1] - P[1], c[2] - P[2]))
    g = tuple(_gap(l[k], H[k]) for k in range(3))
    return dot(g, g) <= r * r


def _sphere_sphere(c, r, P, rc):
    d = (c[0] - P[0], c[1] - P[1], c[2] - P[2])
    return dot(d, d) <= (r + rc) * (r + rc)


def _box_box(c, Qq, H, P, Q, h):
    m = len(P[0])
    one = lambda x: np.full(m, x, np.float32)
    u = [tuple(one(x) for x in qrot(tuple(f(x) for x in Qq), e)) for e in _E]
    v = [qrot(Q, tuple(one(x) for x in e)) for e in _E]
    t = (P[0] - c[0], P[1] - c[1], P[2] - c[2])
    Hs = tuple(f(x) for x in H)

    def radius(hh, a, L):
        return (np.abs(hh[0] * dot(a[0], L)) + np.abs(hh[1] * dot(a[1], L))) + np.abs(hh[2] * dot(a[2], L))

    sep = np.zeros(m, bool)
    axes = u + v + [cross(u[i], v[k]) for i in range(3) for k in range(3)]
    for L in axes:
        sep |= np.abs(dot(t, L)) > radius(Hs, u, L) + radius(h, v, L)
    return ~sep


def _valid(q):
    shape = int(q["shape"])
    c = q["center"]
    if shape == abi.OVERLAP_SPHERE:
        return bool(np.isfinite(c).all() and np.isfinite(q["radius"]) and q["radius"] >= 0)
    if shape == abi.OVERLAP_BOX:
        r, H = q["rotation"].astype(np.float32), q["half_extents"]
        qq = ((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2]) + r[3] * r[3]
        return bool(np.isfinite(c).all() and np.isfinite(r).all() and np.isfinite(H).all() and (H >= 0).all() and qq != 0)
    return False


def query(scene, queries, flags=0):
    """(offsets, hits) for abi.OVERLAP_QUERY rows, by brute force: hits ordered by query, then collider."""
    queries = np.asarray(queries, abi.OVERLAP_QUERY).reshape(-1)
    S = scene
    k = len(S.body)
    idx_all = np.arange(k)
    offsets = np.zeros(len(queries) + 1, np.uint32)
    parts = []
    PW = S.world["position"]; QW = S.world["rotation"]
    with np.errstate(all="ignore"):
        for n, q in enumerate(queries):
            offsets[n] = sum(len(p) for p in parts)
            if not k or not _valid(q):
                continue
            ok = ((S.category & np.uint32(q["mask"])) != 0) & (S.body != q["ignore_body"])
            if not flags & abi.OVERLAP_SENSORS:
                ok &= ~S.sensor
            box = int(q["shape"]) == abi.OVERLAP_BOX
            c = tuple(f(x) for x in q["center"])
            c64 = np.array(c, np.float64)
            rot = q["rotation"].astype(np.float64)
            if box and abs(float(rot @ rot) - 1.0) > 2.0 ** -10:
                reach = np.full(k, np.inf)
            else:
                reach = float(np.linalg.norm(q["half_extents"].astype(np.float64))) if box else float(q["radius"])
                reach = (reach + S.radius64) * (1 + 1e-3) + 1e-4 * (1.0 + np.abs(c64).max() + np.abs(S.p64).max(axis=1))
            ok &= np.linalg.norm(S.p64 - c64, axis=1) <= reach
            cand = idx_all[ok]
            if not len(cand):
                continue
            isbox = cand < S.nboxes
            hit = np.zeros(len(cand), bool)
            P, Qc, H = PW[cand], QW[cand], S.half[cand]
            b, s = isbox, ~isbox
            if box:
                Qq, Hq = q["rotation"].astype(np.float32), q["half_extents"].astype(np.float32)
                if b.any():
                    hit[b] = _box_box(c, Qq, Hq, _cols(P[b]), _cols(Qc[b]), _cols(H[b]))
                if s.any():   # the sphere collider's centre against the query box
                    m = int(s.sum())
                    full = lambda x: np.full(m, x, np.float32)
                    hit[s] = _sphere_box(_cols(P[s]), H[s, 0], tuple(full(x) for x in c), tuple(full(x) for x in Qq), tuple(full(x) for x in Hq))
            else:
                r = f(q["radius"])
                if b.any():
                    hit[b] = _sphere_box(c, r, _cols(P[b]), _cols(Qc[b]), _cols(H[b]))
                if s.any():
                    hit[s] = _sphere_sphere(c, r, _cols(P[s]), H[s, 0])
            got = cand[hit]
            h = np.zeros(len(got), abi.OVERLAP_HIT)
            h["query"] = n; h["collider"] = got; h["body"] = S.body[got]; h["tag"] = S.tag[got]
            parts.append(h)
    hits = np.concatenate(parts) if parts else np.zeros(0, abi.OVERLAP_HIT)
    offsets[len(queries)] = len(hits)
    return offsets, hits
