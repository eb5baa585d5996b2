"""CPU restatement of nb_raycast (nudge_b200/csrc/nb_query_api.cuh) by brute force over every collider — TEST INFRASTRUCTURE ONLY.

The reference has no scene queries.  This follows the float32 arithmetic include/nudge_b200.h states for nb_raycast, operation by
operation (numpy float32 ufuncs round every operation and never fuse), vectorised over the colliders of one ray.  Before the exact
arithmetic a float64 test drops the colliders whose bounding sphere, widened by a relative margin far above float32 rounding, the ray
segment cannot reach; whether and where a collider is hit is decided by the exact arithmetic alone.  The collider world transforms restate
k_collider_world with joints_ref's qrot / qmul."""
import numpy as np
from nudge_b200 import abi, scenes
from oracle.joints_ref import qrot, qmul

f = np.float32
NO_HIT = abi.RAY_NO_HIT


def _cols(a):
    return tuple(a[:, k] for k in range(a.shape[1]))


def world_transforms(body_xf, box_xf, sphere_xf):
    """The world transform of every collider, boxes then spheres, as scenes.TRANSFORM rows (k_collider_world: p = qrot(q_body, p_col) + p_body,
    q = qmul(q_body, q_col), body in the body field)."""
    col = np.concatenate([box_xf, sphere_xf])
    b = body_xf[col["body"].astype(np.int64)]
    bq = _cols(b["rotation"])
    p = qrot(bq, _cols(col["position"]))
    p = (p[0] + b["position"][:, 0], p[1] + b["position"][:, 1], p[2] + b["position"][:, 2])
    q = qmul(bq, _cols(col["rotation"]))
    out = np.zeros(len(col), scenes.TRANSFORM)
    out["position"] = np.stack(p, axis=1); out["rotation"] = np.stack(q, axis=1); out["body"] = col["body"]
    return out


class Scene:
    """The colliders a ray sees: world transforms, shapes, bodies, tags, categories and sensor flags, by collider index."""

    def __init__(self, body_xf, box_xf, box_data, box_tags, sphere_xf, sphere_data, sphere_tags, filters=None, sensors=None):
        self.world = world_transforms(body_xf, box_xf, sphere_xf)
        self.nboxes = len(box_xf)
        self.half = np.concatenate([box_data["size"], np.repeat(sphere_data["radius"][:, None], 3, axis=1)]).astype(np.float32)
        self.body = self.world["body"].copy()
        self.tag = np.concatenate([box_tags, sphere_tags]).astype(np.uint32)
        k = len(self.body)
        self.category = np.full(k, 0xffff, np.uint32) if filters is None else np.asarray(filters["category"], np.uint32)
        self.sensor = np.zeros(k, bool) if sensors is None else np.asarray(sensors) != 0
        self.p64 = self.world["position"].astype(np.float64)
        h = self.half.astype(np.float64)
        self.radius64 = np.where(np.arange(k) < self.nboxes, np.sqrt((h * h).sum(axis=1)), h[:, 0])

    @classmethod
    def of_sim(cls, sim, filters=None, sensors=None):
        """From a Sim's host mirrors (download_bodies() first for the device's transforms)."""
        return cls(sim.transforms, sim.box_transforms, sim.box_data, sim.box_tags, sim.sphere_transforms, sim.sphere_data, sim.sphere_tags, filters, sensors)


def _box(o, d, max_t, P, Q, H):
    """(hit, t, normal) of the header's box test for arrays of boxes."""
    m = len(P)
    qc = (-Q[:, 0], -Q[:, 1], -Q[:, 2], Q[:, 3])
    lo = qrot(qc, (o[0] - P[:, 0], o[1] - P[:, 1], o[2] - P[:, 2]))
    ld = qrot(qc, tuple(np.full(m, d[k], np.float32) for k in range(3)))
    enter, exit_ = np.zeros(m, np.float32), np.full(m, max_t, np.float32)
    axis, s, alive = np.full(m, -1), np.zeros(m, np.float32), np.ones(m, bool)
    for k in range(3):
        z = ld[k] == 0
        alive &= ~(z & ((lo[k] < -H[:, k]) | (lo[k] > H[:, k])))
        t1 = (-H[:, k] - lo[k]) / ld[k]; t2 = (H[:, k] - lo[k]) / ld[k]
        lt = t1 < t2
        near, far = np.where(lt, t1, t2), np.where(lt, t2, t1)
        up = ~z & (near > enter)
        enter = np.where(up, near, enter); axis = np.where(up, k, axis); s = np.where(up, np.where(lt, f(-1.0), f(1.0)), s)
        exit_ = np.where(~z & (far < exit_), far, exit_)
        alive &= ~(~z & (enter > exit_))
    zero = np.zeros(m, np.float32)
    nl = tuple(np.where(axis == k, s, zero) for k in range(3))
    n = qrot(tuple(Q[:, k] for k in range(4)), nl)
    n = np.stack([np.where(axis < 0, zero, c) for c in n], axis=1)
    return alive, enter, n


def _sphere(o, d, max_t, P, r):
    m = (o[0] - P[:, 0], o[1] - P[:, 1], o[2] - P[:, 2])
    a = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
    b = (m[0] * d[0] + m[1] * d[1]) + m[2] * d[2]
    c = ((m[0] * m[0] + m[1] * m[1]) + m[2] * m[2]) - r * r
    inside = c <= 0
    disc = b * b - a * c
    t = (-b - np.sqrt(disc)) / a
    hit = inside | (~(disc < 0) & (t >= 0) & (t <= max_t))
    t = np.where(inside, f(0.0), t)
    t = np.where(t == 0, f(0.0), t)
    inv = f(1.0) / r
    pos = [o[k] + t * d[k] for k in range(3)]
    n = np.stack([(pos[k] - P[:, k]) * inv for k in range(3)], axis=1)
    n = np.where(inside[:, None], f(0.0), n)
    return hit, t, n


def _valid(ray):
    o, d, mt = ray["origin"], ray["direction"], ray["max_t"]
    return bool(np.isfinite(o).all() and np.isfinite(d).all() and np.isfinite(mt) and mt >= 0 and (d != 0).any())


def cast(scene, rays, flags=0):
    """abi.RAY_HIT rows for abi.RAY rows, by brute force."""
    rays = np.asarray(rays, abi.RAY).reshape(-1)
    out = np.zeros(len(rays), abi.RAY_HIT)
    out["collider"] = out["body"] = out["tag"] = NO_HIT
    S = scene
    idx_all = np.arange(len(S.body))
    with np.errstate(all="ignore"):
        for n, ray in enumerate(rays):
            if not _valid(ray) or not len(S.body):
                continue
            o, d, max_t = tuple(f(x) for x in ray["origin"]), tuple(f(x) for x in ray["direction"]), f(ray["max_t"])
            ok = ((S.category & np.uint32(ray["mask"])) != 0) & (S.body != ray["ignore_body"])
            if not flags & abi.RAY_SENSORS:
                ok &= ~S.sensor
            # float64 reach test: the bounding sphere against the segment [0, max_t], widened
            o64, d64 = np.array(o, np.float64), np.array(d, np.float64)
            w = S.p64 - o64
            tp = np.clip(w @ d64 / (d64 @ d64), 0.0, float(max_t))
            dist = np.linalg.norm(w - tp[:, None] * d64[None, :], axis=1)
            # the sphere test's disc = b*b - a*c cancels, so the stated arithmetic can hit about 2^-10.5 |o - p| outside a sphere: 2^-8 of it
            ok &= dist <= S.radius64 * (1 + 1e-4) + 1e-4 * (1.0 + np.abs(o64).max() + 2.0 * np.abs(S.p64).max(axis=1) + S.radius64) + \
                np.linalg.norm(w, axis=1) / 256.0
            cand = idx_all[ok]
            if not len(cand):
                continue
            P, Q, H = S.world["position"][cand], S.world["rotation"][cand], S.half[cand]
            isbox = cand < S.nboxes
            hit, t, nrm = np.zeros(len(cand), bool), np.zeros(len(cand), np.float32), np.zeros((len(cand), 3), np.float32)
            if isbox.any():
                hit[isbox], t[isbox], nrm[isbox] = _box(o, d, max_t, P[isbox], Q[isbox], H[isbox])
            if (~isbox).any():
                hit[~isbox], t[~isbox], nrm[~isbox] = _sphere(o, d, max_t, P[~isbox], H[~isbox, 0])
            if not hit.any():
                continue
            keys = (t.view(np.uint32).astype(np.uint64) << np.uint64(32)) | cand.astype(np.uint64)
            keys[~hit] = np.uint64(0xffffffffffffffff)
            w_ = int(np.argmin(keys))
            tt, i = t[w_], int(cand[w_])
            h = out[n]
            h["t"] = tt
            h["position"] = [o[k] + tt * d[k] for k in range(3)]
            h["normal"] = nrm[w_]
            h["collider"], h["body"], h["tag"] = i, S.body[i], S.tag[i]
    return out
